#include "client.h"

#include <errno.h>
#include <poll.h>
#include <sys/socket.h>

#include <errno.h>
#include <fcntl.h>
#include <sys/vfs.h>
#include <unistd.h>

#include <algorithm>
#include <fstream>
#include <random>
#include <sstream>

#include "net.h"

namespace cv {

// ------------------------------------------------------------------ FileBlocks / Namespace

void FileBlocks::build_index() {
    starts.clear();
    int64_t off = 0;
    for (const auto& b : block_locs) {
        starts.push_back(off);
        off += b.block.len;
    }
}

Err FileBlocks::get_read_block(int64_t pos, int64_t* block_off, size_t* index) const {
    // partition_point(|x| x.end <= pos)
    size_t lo = 0, hi = block_locs.size();
    while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        if (starts[mid] + block_locs[mid].block.len <= pos) lo = mid + 1;
        else hi = mid;
    }
    if (lo >= block_locs.size()) return Err::common(str_printf("Not found block for pos %lld", (long long)pos));
    *block_off = pos - starts[lo];
    *index = lo;
    return Err::ok();
}

Err Namespace::load(const std::string& path) {
    std::ifstream f(path);
    if (!f) return Err(kFileNotFound, "namespace manifest not found: " + path);
    std::stringstream ss;
    ss << f.rdbuf();
    return load_string(ss.str());
}

// manifest lines:
//   file  <path> <inode_id> <len> <block_size> <mtime>
//   block <block_id> <len> <storage_type> <crc32 hex|-> <crc32c hex|-> <h|-> <host:port:worker_id,...|->
Err Namespace::load_string(const std::string& text) {
    std::istringstream in(text);
    std::string line;
    FileBlocks cur;
    bool have = false;
    auto flush = [&] {
        if (have) {
            cur.build_index();
            put(cur);
        }
        have = false;
    };
    while (std::getline(in, line)) {
        if (line.empty() || line[0] == '#') continue;
        std::istringstream ls(line);
        std::string kind;
        ls >> kind;
        if (kind == "file") {
            flush();
            cur = FileBlocks();
            ls >> cur.status.path >> cur.status.id >> cur.status.len >> cur.status.block_size >> cur.status.mtime;
            if (ls.fail()) return Err::common("bad manifest line: " + line);
            have = true;
        } else if (kind == "block") {
            if (!have) return Err::common("manifest: block before file");
            LocatedBlock lb;
            std::string c32, c32c, flags, locs;
            ls >> lb.block.id >> lb.block.len >> lb.block.storage_type >> c32 >> c32c >> flags >> locs;
            if (ls.fail()) return Err::common("bad manifest line: " + line);
            if (c32 != "-" && c32c != "-") {
                lb.crc32 = static_cast<uint32_t>(strtoul(c32.c_str(), nullptr, 16));
                lb.crc32c = static_cast<uint32_t>(strtoul(c32c.c_str(), nullptr, 16));
                lb.has_crc = true;
            }
            lb.block.has_alloc_opts = flags.find('h') != std::string::npos;
            if (locs != "-") {
                std::istringstream lss(locs);
                std::string one;
                while (std::getline(lss, one, ',')) {
                    WorkerAddress a;
                    const size_t c1 = one.find(':'), c2 = one.find(':', c1 + 1);
                    if (c1 == std::string::npos) return Err::common("bad worker address: " + one);
                    a.hostname = a.ip_addr = one.substr(0, c1);
                    a.rpc_port = static_cast<uint32_t>(atoi(one.substr(c1 + 1, c2 == std::string::npos ? std::string::npos : c2 - c1 - 1).c_str()));
                    if (c2 != std::string::npos) a.worker_id = static_cast<uint32_t>(atoi(one.substr(c2 + 1).c_str()));
                    lb.locs.push_back(a);
                }
            }
            cur.block_locs.push_back(lb);
        } else {
            return Err::common("bad manifest line: " + line);
        }
    }
    flush();
    return Err::ok();
}

std::string Namespace::dump() const {
    std::lock_guard<std::mutex> lk(mu_);
    std::string out = "# curvine-b200 namespace manifest v1\n";
    for (const auto& kv : files_) {
        const FileBlocks& f = *kv.second;
        out += str_printf("file %s %lld %lld %lld %lld\n", f.status.path.c_str(), (long long)f.status.id, (long long)f.status.len,
                          (long long)f.status.block_size, (long long)f.status.mtime);
        for (const auto& b : f.block_locs) {
            std::string locs;
            for (const auto& a : b.locs) locs += (locs.empty() ? "" : ",") + a.hostname + ":" + std::to_string(a.rpc_port) + ":" + std::to_string(a.worker_id);
            if (locs.empty()) locs = "-";
            const std::string c1 = b.has_crc ? str_printf("%08x", b.crc32) : "-", c2 = b.has_crc ? str_printf("%08x", b.crc32c) : "-";
            out += str_printf("block %lld %lld %d %s %s %s %s\n", (long long)b.block.id, (long long)b.block.len, b.block.storage_type, c1.c_str(),
                              c2.c_str(), b.block.has_alloc_opts ? "h" : "-", locs.c_str());
        }
    }
    return out;
}

void Namespace::put(const FileBlocks& fb) {
    std::shared_ptr<FileBlocks> c(new FileBlocks(fb));
    c->build_index();
    std::lock_guard<std::mutex> lk(mu_);
    files_[fb.status.path] = std::move(c);
}

Err Namespace::get_block_locations(const std::string& path, std::shared_ptr<const FileBlocks>* out) const {
    std::lock_guard<std::mutex> lk(mu_);
    auto it = files_.find(path);
    if (it == files_.end()) return Err(kFileNotFound, "File " + path + " not exists");
    *out = it->second;
    return Err::ok();
}

// ------------------------------------------------------------------ BlockClient

BlockClient::~BlockClient() { close_fd(fd_); }

Err BlockClient::drain_pending() {
    Protocol resp;
    std::string rh, rd;
    while (!pending_.empty()) {
        const Protocol req = pending_.front();
        pending_.erase(pending_.begin());
        CV_RETURN_IF_ERR(recv_answer(req, &resp, &rh, &rd));
    }
    return Err::ok();
}

void BlockClient::append_frame(const Protocol& req, const std::string& header, std::string* out, int32_t data_len) {
    Protocol p = req;
    p.header_len = static_cast<int32_t>(header.size()), p.data_len = data_len;
    const size_t at = out->size();
    out->resize(at + kProtocolSize);
    encode_protocol(p, reinterpret_cast<uint8_t*>(&(*out)[at]));
    out->append(header);
}

Err BlockClient::send_request(const Protocol& req, const std::string& header) {
    CV_RETURN_IF_ERR(drain_pending());
    std::string out;
    append_frame(req, header, &out);
    Err e = send_all(fd_, out.data(), out.size());
    if (e) broken = true;
    return e;
}

Err BlockClient::recv_answer(const Protocol& req, Protocol* resp, std::string* header, std::string* data) {
    uint8_t prefix[kProtocolSize];
    Err e;
    do {  // heartbeats are read whole and skipped (rpc_frame.rs:255-259)
        e = recv_exact(fd_, prefix, kProtocolSize);
        if (!e) e = decode_protocol(prefix, resp);
        if (!e && resp->header_len < 0) e = Err::common(str_printf("Invalid length %d", resp->header_len));
        if (e) break;
        header->resize(static_cast<size_t>(resp->header_len));
        data->resize(static_cast<size_t>(resp->data_len));
        if (resp->header_len) e = recv_exact(fd_, &(*header)[0], header->size());
        if (!e && resp->data_len) e = recv_exact(fd_, &(*data)[0], data->size());
    } while (!e && resp->is_heartbeat());
    if (!e && (req.req_id != resp->req_id || req.seq_id != resp->seq_id))  // raw_client.rs:100-116
        e = Err::common(str_printf("response mismatch: request (req_id %lld, seq_id %d), response (req_id %lld, seq_id %d)", (long long)req.req_id,
                                   req.seq_id, (long long)resp->req_id, resp->seq_id));
    if (e) {
        broken = true;
        return e;
    }
    return resp->is_success() ? Err::ok() : decode_error_body(reinterpret_cast<const uint8_t*>(data->data()), data->size());
}

Err BlockClient::rpc(const Protocol& req, const std::string& header, Protocol* resp, std::string* resp_header, std::string* resp_data) {
    CV_RETURN_IF_ERR(send_request(req, header));
    return recv_answer(req, resp, resp_header, resp_data);
}

static BlockReadRequest open_request(const ClientConf& conf, const ExtendedBlock& b, int64_t off, int64_t len, bool short_circuit, int64_t chunk_size,
                                     bool accept_arena) {
    BlockReadRequest r;
    r.id = b.id, r.off = off, r.len = len, r.chunk_size = static_cast<int32_t>(chunk_size), r.short_circuit = short_circuit;
    r.accept_arena = accept_arena && short_circuit;
    r.enable_read_ahead = conf.enable_read_ahead, r.read_ahead_len = conf.read_ahead_len, r.drop_cache_len = conf.drop_cache_len;
    return r;
}

Err BlockClient::open_block(const ClientConf& conf, const ExtendedBlock& b, int64_t off, int64_t len, int64_t req_id, int32_t seq_id,
                            bool short_circuit, int64_t chunk_size, BlockReadResponse* out, bool accept_arena) {
    const BlockReadRequest r = open_request(conf, b, off, len, short_circuit, chunk_size, accept_arena);
    Protocol resp;
    std::string rh, rd;
    CV_RETURN_IF_ERR(rpc(request_proto(kCodeReadBlock, kReqOpen, req_id, seq_id), r.encode(), &resp, &rh, &rd));
    return BlockReadResponse::decode(reinterpret_cast<const uint8_t*>(rh.data()), rh.size(), out);
}

Err BlockClient::read_commit(const ExtendedBlock& b, int64_t req_id, int32_t seq_id) {
    BlockReadRequest r;  // ..Default::default(): proto defaults for everything but id (block_client.rs:263-266)
    r.id = b.id;
    Protocol resp;
    std::string rh, rd;
    return rpc(request_proto(kCodeReadBlock, kReqComplete, req_id, seq_id), r.encode(), &resp, &rh, &rd);
}

Err BlockClient::read_commit_deferred(const ExtendedBlock& b, int64_t req_id, int32_t seq_id) {
    BlockReadRequest r;
    r.id = b.id;
    const Protocol p = request_proto(kCodeReadBlock, kReqComplete, req_id, seq_id);
    CV_RETURN_IF_ERR(send_request(p, r.encode()));
    pending_.push_back(p);
    return Err::ok();
}

Err BlockClient::open_blocks(const ClientConf& conf, const std::vector<OpenReq>& reqs, int64_t chunk_size, bool accept_arena,
                             std::vector<BlockReadResponse>* out) {
    std::string buf;
    for (const OpenReq& q : reqs)
        append_frame(request_proto(kCodeReadBlock, kReqOpen, q.req_id, 0), open_request(conf, *q.b, q.off, q.b->len, true, chunk_size, accept_arena).encode(), &buf);
    Err e = send_all(fd_, buf.data(), buf.size());
    if (!e) e = drain_pending();  // the worker answers in order: the deferred Completes' answers come first
    out->assign(reqs.size(), BlockReadResponse());
    Protocol resp;
    std::string rh, rd;
    for (size_t i = 0; i < reqs.size() && !e; i++) {
        e = recv_answer(request_proto(kCodeReadBlock, kReqOpen, reqs[i].req_id, 0), &resp, &rh, &rd);
        if (!e) e = BlockReadResponse::decode(reinterpret_cast<const uint8_t*>(rh.data()), rh.size(), &(*out)[i]);
    }
    if (e) broken = true;
    return e;
}

Err BlockClient::read_commit_deferred(const std::vector<OpenReq>& reqs) {
    std::string buf;
    for (const OpenReq& q : reqs) {
        BlockReadRequest r;
        r.id = q.b->id;
        append_frame(request_proto(kCodeReadBlock, kReqComplete, q.req_id, 1), r.encode(), &buf);
    }
    if (Err e = send_all(fd_, buf.data(), buf.size())) {
        broken = true;
        return e;
    }
    for (const OpenReq& q : reqs) pending_.push_back(request_proto(kCodeReadBlock, kReqComplete, q.req_id, 1));
    return Err::ok();
}

Err BlockClient::send_block_read_pipeline(const ClientConf& conf, const ExtendedBlock& b, int64_t off, int64_t req_id, int64_t chunk_size, int64_t n_running,
                                          BlockReadResponse* open_resp) {
    CV_RETURN_IF_ERR(drain_pending());
    const BlockReadRequest r = open_request(conf, b, off, b.len, false, chunk_size, false);
    std::string out;
    const Protocol open = request_proto(kCodeReadBlock, kReqOpen, req_id, 0);
    append_frame(open, r.encode(), &out);
    for (int64_t f = 0; f < n_running; f++) append_frame(request_proto(kCodeReadBlock, kReqRunning, req_id, static_cast<int32_t>(f + 1)), std::string(), &out);
    BlockReadRequest c;  // ..Default::default() but the id (block_client.rs:263-266)
    c.id = b.id;
    const Protocol complete = request_proto(kCodeReadBlock, kReqComplete, req_id, static_cast<int32_t>(n_running + 1));
    append_frame(complete, c.encode(), &out);
    Protocol resp;
    std::string rh, rd;
    Err e = send_all(fd_, out.data(), out.size());
    if (!e) e = recv_answer(open, &resp, &rh, &rd);
    if (!e) e = BlockReadResponse::decode(reinterpret_cast<const uint8_t*>(rh.data()), rh.size(), open_resp);
    if (e) {
        broken = true;  // the answers to the requests already sent behind the Open are dropped with the connection
        return e;
    }
    pending_.push_back(complete);
    return Err::ok();
}

// ------------------------------------------------------------------ FsContext (connection pool)

FsContext::~FsContext() = default;

static int64_t now_ms() { return static_cast<int64_t>(now_sec() * 1000.0); }

// A pooled connection whose peer went away (worker restarted, idle timeout on the server side) has a FIN or RST queued: a
// non-blocking peek sees it without consuming anything.  An idle healthy connection has nothing to read (EAGAIN); bytes nobody
// asked for mean the stream is out of step.  Either way the connection is not handed out again.
static bool pooled_connection_is_usable(int fd, bool answers_outstanding = false) {
    // the peer's hang-up first: a worker that answered a parked deferred Complete and then went away leaves DATA and the FIN in the socket, and
    // a peek alone would see only the data
    struct pollfd p;
    p.fd = fd, p.events = POLLIN | POLLRDHUP, p.revents = 0;
    if (::poll(&p, 1, 0) < 0 || (p.revents & (POLLRDHUP | POLLHUP | POLLERR | POLLNVAL))) return false;
    char b;
    const ssize_t r = ::recv(fd, &b, 1, MSG_PEEK | MSG_DONTWAIT);
    if (r < 0 && (errno == EAGAIN || errno == EWOULDBLOCK)) return true;
    return answers_outstanding && r > 0;  // a parked deferred Complete: its answer may already sit in the socket; EOF / RST still disqualify
}

Err FsContext::acquire_read(const WorkerAddress& addr, std::unique_ptr<BlockClient>* out) {
    if (conf.client.enable_block_conn_pool) {
        std::vector<std::unique_ptr<BlockClient>> expired;  // closed outside the lock
        std::lock_guard<std::mutex> lk(mu_);
        auto& v = idle_[addr.str()];
        const int64_t now = now_ms();
        while (!v.empty()) {
            std::unique_ptr<BlockClient> c = std::move(v.back());  // LIFO
            v.pop_back();
            idle_total_--;
            // a connection parked with a deferred Complete outstanding has (or will have) that response queued: it is consumed by
            // the next request, so readable bytes are expected on it
            if (now - c->idle_since_ms < conf.client.block_conn_idle_time_ms && pooled_connection_is_usable(c->fd(), c->pending() > 0)) {
                *out = std::move(c);
                return Err::ok();
            }
            expired.push_back(std::move(c));
            conns_expired_++;
        }
    }
    int fd = -1;
    if (conf.b200.socket_buffer > 0) set_socket_buffer_bytes(static_cast<int>(std::min<int64_t>(conf.b200.socket_buffer, 1 << 30)));
    // a worker on this host: its abstract unix socket first when configured (same frames, less protocol work per byte)
    if (!(conf.b200.local_unix_socket && is_local_worker(addr) && !unix_connect(local_socket_name(static_cast<int>(addr.rpc_port)), &fd, conf.client.data_timeout_ms)))
        CV_RETURN_IF_ERR(tcp_connect(addr.ip_addr.empty() ? addr.hostname : addr.ip_addr, static_cast<int>(addr.rpc_port), &fd, conf.client.conn_timeout_ms,
                                     conf.client.data_timeout_ms));
    out->reset(new BlockClient(fd, addr));
    {
        std::lock_guard<std::mutex> lk(mu_);
        conns_opened_++;
    }
    return Err::ok();
}

void FsContext::release(std::unique_ptr<BlockClient> c) {
    if (!c || c->broken || !conf.client.enable_block_conn_pool) return;
    std::lock_guard<std::mutex> lk(mu_);
    if (idle_total_ >= conf.client.block_conn_idle_size) return;  // pool full: the connection is closed
    c->idle_since_ms = now_ms();
    idle_[c->addr().str()].push_back(std::move(c));
    idle_total_++;
}

Err FsContext::connection_to(const WorkerAddress& addr, std::unique_ptr<BlockClient>* conn) {
    if (*conn && (*conn)->addr() == addr && !(*conn)->broken) return Err::ok();
    release(std::move(*conn));
    return acquire_read(addr, conn);
}

void FsContext::add_failed_worker(const WorkerAddress& addr) {
    std::lock_guard<std::mutex> lk(fw_mu_);
    failed_workers_[addr.worker_id] = now_ms() + conf.client.failed_worker_ttl_ms;
}

std::vector<uint32_t> FsContext::get_failed_workers() {
    std::vector<uint32_t> out;
    std::lock_guard<std::mutex> lk(fw_mu_);
    const int64_t now = now_ms();
    for (auto it = failed_workers_.begin(); it != failed_workers_.end();) {
        if (it->second <= now) it = failed_workers_.erase(it);  // time_to_live elapsed
        else out.push_back((it++)->first);
    }
    std::sort(out.begin(), out.end());
    return out;
}

bool FsContext::is_failed_worker(const WorkerAddress& addr) {
    for (uint32_t id : get_failed_workers())
        if (id == addr.worker_id) return true;
    return false;
}

Err FsContext::no_available_worker(const std::vector<WorkerAddress>& locs) {
    std::string l, f;
    for (const auto& a : locs) l += (l.empty() ? "" : ", ") + a.str();
    for (uint32_t id : get_failed_workers()) f += (f.empty() ? "" : ", ") + std::to_string(id);
    return Err::common("There is no available worker, locs: [" + l + "], failed workers: [" + f + "]");
}

void FsContext::pool_stats(int64_t out[3]) {
    std::lock_guard<std::mutex> lk(mu_);
    out[0] = idle_total_, out[1] = conns_opened_, out[2] = conns_expired_;
}

// ------------------------------------------------------------------ BlockReader

BlockReader::~BlockReader() { drop_adapter(); }

void BlockReader::drop_adapter() {
    close_fd(fd_);
    fd_ = -1;
    if (client_) ctx_->release(std::move(client_));
}

Err BlockReader::create(FsContext* ctx, const LocatedBlock& lb, int64_t off, std::unique_ptr<BlockReader>* out) {
    std::unique_ptr<BlockReader> r(new BlockReader());
    r->ctx_ = ctx;
    r->block_ = lb.block;
    r->chunk_size_ = ctx->read_chunk_size();
    r->locs_ = lb.locs;
    // sort_locs (block_reader.rs:146-166): shuffle, then the local worker first when short-circuit is on
    if (r->locs_.size() > 1) {
        static thread_local std::mt19937 rng{std::random_device{}()};
        std::shuffle(r->locs_.begin(), r->locs_.end(), rng);
    }
    if (ctx->conf.client.short_circuit)
        for (size_t i = 0; i < r->locs_.size(); i++)
            if (ctx->is_local_worker(r->locs_[i])) {
                std::swap(r->locs_[0], r->locs_[i]);
                break;
            }
    CV_RETURN_IF_ERR(r->open_adapter(off));
    *out = std::move(r);
    return Err::ok();
}

// BlockReader::get_reader (block_reader.rs:168-215).  As in the reference, the `?` on the adapter constructors
// propagates the first candidate's open error out of the function: there is no open-time failover, only the
// read-time failover in read().
Err BlockReader::open_adapter(int64_t off) {
    drop_adapter();
    pos_ = off;
    if (locs_.empty() && block_.has_alloc_opts) {
        kind_ = kHole;
        cur_addr_ = WorkerAddress();
        return Err::ok();
    }
    if (locs_.empty()) return ctx_->no_available_worker(locs_);
    const WorkerAddress& loc = locs_[0];
    cur_addr_ = loc;
    const bool sc = ctx_->conf.client.short_circuit && ctx_->is_local_worker(loc);
    req_id_ = new_req_id();
    seq_id_ = 0;
    pending_seek_ = false;
    CV_RETURN_IF_ERR(ctx_->acquire_read(loc, &client_));
    BlockReadResponse resp;
    Err e = client_->open_block(ctx_->conf.client, block_, off, block_.len, req_id_, seq_id_, sc, chunk_size_, &resp, ctx_->conf.b200.arena);
    if (e) {
        drop_adapter();
        return e;
    }
    if (sc) {
        if (!resp.has_path) {
            drop_adapter();
            return Err::common("read_context.path is none");
        }
        fd_ = ::open(resp.path.c_str(), O_RDONLY | O_CLOEXEC);
        if (fd_ < 0) {
            drop_adapter();
            return Err::io(str_printf("open %s: %s", resp.path.c_str(), strerror(errno)));
        }
        ctx_->release(std::move(client_));  // BlockReaderLocal keeps no connection; complete() acquires a new one
        kind_ = kLocal;
        base_off_ = resp.has_arena ? resp.arena_off : 0;  // arena block: the bytes start at arena_off inside the segment file
        struct statfs sfs;
        const bool tmpfs = fstatfs(fd_, &sfs) == 0 && sfs.f_type == 0x01021994;  // sys_libc.rs:320-339
        ra_enabled_ = ctx_->conf.client.enable_read_ahead && !tmpfs && block_.len >= 256 * 1024;
        last_ahead_ = -1;
    } else {
        kind_ = kRemote;
    }
    return Err::ok();
}

Err BlockReader::seek(int64_t pos) {
    pos_ = pos;
    if (kind_ == kRemote) pending_seek_ = true;  // piggy-backed on the next Running request (block_reader_remote.rs:93-101)
    return Err::ok();
}

Err BlockReader::read_once(std::string* buf) {
    if (remaining() <= 0) return Err::common("No readable data");
    const int64_t want = std::min<int64_t>(chunk_size_, remaining());
    switch (kind_) {
        case kHole:
            buf->assign(static_cast<size_t>(want), '\0');
            break;
        case kLocal: {
            // CacheManager::read_ahead (orpc/src/sys/cache_manager.rs:99-147, block_reader_local.rs:113-126): hint the next
            // read_ahead_len bytes once the cursor passed half of the previous window; never on tmpfs or small files
            if (ra_enabled_ && (last_ahead_ < 0 || pos_ >= last_ahead_ + ctx_->conf.client.read_ahead_len / 2)) {
                posix_fadvise(fd_, base_off_ + pos_, ctx_->conf.client.read_ahead_len, POSIX_FADV_WILLNEED);
                last_ahead_ = pos_;
            }
            if (buf->size() != static_cast<size_t>(want)) buf->resize(static_cast<size_t>(want));  // a recycled chunk buffer of the same size is not zero-filled again (the reference's BytesMut is not either: rpc_frame.rs set_len)
            int64_t got = 0;
            while (got < want) {
                const ssize_t r = pread(fd_, &(*buf)[got], static_cast<size_t>(want - got), base_off_ + pos_ + got);
                if (r < 0 && errno == EINTR) continue;
                if (r <= 0) return Err::io(str_printf("read block file: %s", r == 0 ? "unexpected eof" : strerror(errno)));
                got += r;
            }
            break;
        }
        case kRemote: {
            std::string header;
            if (pending_seek_) {
                DataHeaderProto h;
                h.offset = pos_;
                header = h.encode();
                pending_seek_ = false;
            }
            Protocol resp;
            std::string rh;
            CV_RETURN_IF_ERR(client_->rpc(request_proto(kCodeReadBlock, kReqRunning, req_id_, ++seq_id_), header, &resp, &rh, buf));
            break;
        }
    }
    pos_ += static_cast<int64_t>(buf->size());
    return Err::ok();
}

// `buf` may arrive holding a previous chunk (its storage is reused); it is empty on return at end of block and after an error.
Err BlockReader::read(std::string* buf) {
    if (!has_remaining()) {  // end of block file
        buf->clear();
        return Err::ok();
    }
    for (;;) {
        Err e = read_once(buf);
        if (!e) return e;
        buf->clear();
        if (kind_ == kHole || locs_.empty()) return e.ctx("failed to read block on " + cur_addr_.str());
        // drop this worker, reopen at pos on the next replica (block_reader.rs:223-252)
        locs_.erase(std::remove(locs_.begin(), locs_.end(), cur_addr_), locs_.end());
        if (client_) client_->broken = true;
        CV_RETURN_IF_ERR(open_adapter(pos_));
    }
}

Err BlockReader::complete() {
    Err e;
    if (kind_ == kRemote && client_) {
        e = client_->read_commit(block_, req_id_, ++seq_id_);
    } else if (kind_ == kLocal) {
        std::unique_ptr<BlockClient> c;
        e = ctx_->acquire_read(cur_addr_, &c);
        if (!e) e = c->read_commit(block_, req_id_, ++seq_id_);
        if (c) ctx_->release(std::move(c));
    }
    drop_adapter();
    kind_ = kHole;
    locs_.clear();
    return e;
}

// ------------------------------------------------------------------ split / detector

std::vector<std::vector<std::pair<int64_t, int64_t>>> split_slices(int64_t total, int64_t slice_size, int64_t read_parallel) {
    std::vector<std::vector<std::pair<int64_t, int64_t>>> out;
    if (total <= 0) return out;
    if (read_parallel == 1) {
        out.push_back({{0, total}});
        return out;
    }
    const int64_t num = (total + slice_size - 1) / slice_size;
    out.resize(static_cast<size_t>(read_parallel));
    for (int64_t sid = 0; sid < num; sid++) {
        const int64_t start = sid * slice_size, end = sid == num - 1 ? total : start + slice_size;
        out[static_cast<size_t>(sid % read_parallel)].push_back({start, end});
    }
    return out;
}

ReadDetector::ReadDetector(const ClientConf& conf, int64_t file_size) {
    read_parallel = conf.read_parallel;
    if (conf.enable_smart_prefetch && file_size >= conf.large_file_size) {
        const int64_t calc = (file_size + conf.large_file_size - 1) / conf.large_file_size;
        read_parallel = std::min<int64_t>(conf.max_read_parallel, std::max<int64_t>(1, calc));
    }
    enabled = conf.enable_smart_prefetch;
    threshold_ = static_cast<uint64_t>(conf.sequential_read_threshold);
}

void ReadDetector::record_seek() {
    if (!enabled) return;
    seq_count_ = 0;
    last_read_pos_ = -1;
    random_ = true;
}

bool ReadDetector::record_read(int64_t start, int64_t end) {
    if (!enabled) return false;
    if (last_read_pos_ == -1 || start == last_read_pos_) seq_count_++;
    else seq_count_ = 0;
    last_read_pos_ = end;
    const bool now_random = seq_count_ >= threshold_ ? false : random_;
    if (now_random != random_) {
        random_ = now_random;
        return true;
    }
    return false;
}

// ------------------------------------------------------------------ FsReaderBase / FsReaderParallel

FsReaderBase::FsReaderBase(FsContext* ctx, const FileBlocks* fb, bool cache_handles)
    : ctx_(ctx), fb_(fb), len_(fb->status.len), cache_limit_(cache_handles ? static_cast<size_t>(ctx->conf.client.max_cache_block_handles) : 0) {}

FsReaderBase::~FsReaderBase() = default;

Err FsReaderBase::update_reader(std::unique_ptr<BlockReader> cur, bool cache) {
    std::unique_ptr<BlockReader> old = std::move(cur_);
    cur_ = std::move(cur);
    if (!old) return Err::ok();
    if (cache && cache_limit_ > 0) {
        if (cache_.size() >= cache_limit_) {
            std::unique_ptr<BlockReader> removed = std::move(cache_.front());
            cache_.pop_front();
            CV_RETURN_IF_ERR(removed->complete());
        }
        cache_.push_back(std::move(old));
        return Err::ok();
    }
    return old->complete();
}

Err FsReaderBase::get_reader() {
    if (cur_ && cur_->has_remaining()) return Err::ok();
    int64_t boff;
    size_t idx;
    CV_RETURN_IF_ERR(fb_->get_read_block(pos_, &boff, &idx));
    const LocatedBlock& lb = fb_->block_locs[idx];
    std::unique_ptr<BlockReader> nr;
    for (auto it = cache_.begin(); it != cache_.end(); ++it)
        if ((*it)->block_id() == lb.block.id) {
            nr = std::move(*it);
            cache_.erase(it);
            CV_RETURN_IF_ERR(nr->seek(boff));
            break;
        }
    if (!nr) CV_RETURN_IF_ERR(BlockReader::create(ctx_, lb, boff, &nr));
    return update_reader(std::move(nr), false);
}

Err FsReaderBase::read(std::string* buf) {
    if (pos_ >= len_) {
        buf->clear();
        return Err::ok();
    }
    if (Err e = get_reader()) {
        buf->clear();
        return e;
    }
    CV_RETURN_IF_ERR(cur_->read(buf));
    pos_ += static_cast<int64_t>(buf->size());
    return Err::ok();
}

Err FsReaderBase::seek(int64_t pos) {
    if (pos == pos_) return Err::ok();
    if (pos == len_) {
        pos_ = pos;
        return update_reader(nullptr, false);
    }
    if (pos > len_) return Err::common(str_printf("seek position %lld can not exceed file len %lld", (long long)pos, (long long)len_));
    int64_t boff;
    size_t idx;
    CV_RETURN_IF_ERR(fb_->get_read_block(pos, &boff, &idx));
    if (cur_) {
        if (cur_->block_id() == fb_->block_locs[idx].block.id) CV_RETURN_IF_ERR(cur_->seek(boff));
        else CV_RETURN_IF_ERR(update_reader(nullptr, true));
    }
    pos_ = pos;
    return Err::ok();
}

Err FsReaderBase::complete() {
    Err first;
    if (cur_) {
        Err e = cur_->complete();
        if (e && !first) first = e;
        cur_.reset();
    }
    for (auto& r : cache_) {
        Err e = r->complete();
        if (e && !first) first = e;
    }
    cache_.clear();
    return first;
}

Err FsReaderParallel::read(int64_t* off, std::string* buf) {
    *off = 0;
    Err e;
    bool empty = slices_.empty();
    if (!empty && cur_ < 0) {
        cur_ = 0;
        e = inner_.seek(slices_[0].first);
    } else if (!empty && inner_.pos() >= slices_[static_cast<size_t>(cur_)].second) {
        const int64_t next = cur_ + 1;
        if (next >= static_cast<int64_t>(slices_.size())) empty = true;  // FileChunk::default()
        else {
            cur_ = next;
            e = inner_.seek(slices_[static_cast<size_t>(next)].first);
        }
    }
    if (empty || e) {
        buf->clear();
        return e;
    }
    *off = inner_.pos();
    return inner_.read(buf);
}

Err FsReaderParallel::seek(int64_t pos) {
    // first slice with end > pos
    size_t idx = 0;
    while (idx < slices_.size() && slices_[idx].second <= pos) idx++;
    if (idx < slices_.size()) {
        CV_RETURN_IF_ERR(inner_.seek(std::max(pos, slices_[idx].first)));
        cur_ = static_cast<int64_t>(idx);
    } else if (!slices_.empty()) {
        CV_RETURN_IF_ERR(inner_.seek(slices_.back().second));
        cur_ = static_cast<int64_t>(slices_.size()) - 1;
    } else {
        CV_RETURN_IF_ERR(inner_.seek(0));
        cur_ = -1;
    }
    return Err::ok();
}

// ------------------------------------------------------------------ FsReader

Err FsReader::open(FsContext* ctx, const std::string& path, std::unique_ptr<FsReader>* out) {
    std::unique_ptr<FsReader> r(new FsReader());
    r->ctx_ = ctx;
    CV_RETURN_IF_ERR(ctx->ns.get_block_locations(path, &r->fb_));
    const ClientConf& c = ctx->conf.client;
    r->len_ = r->fb_->status.len;
    r->chunk_size_ = c.read_chunk_size;
    r->slice_size_ = c.read_slice_size;
    r->det_ = ReadDetector(c, r->len_);
    // FsReaderParallel::create_all checks (fs_reader_parallel.rs:62-71)
    if (c.read_chunk_size % 4096 != 0 || c.read_chunk_size < 4096) return Err::common("chunk_size must be an integer multiple of 4096");
    if (r->slice_size_ % c.read_chunk_size != 0 || r->slice_size_ < c.read_chunk_size)
        return Err::common("The slice size must be an integer multiple of the chunk size.");
    for (auto& s : split_slices(r->len_, r->slice_size_, r->det_.read_parallel))
        if (!s.empty()) {
            std::unique_ptr<FsReaderParallel> pr(new FsReaderParallel(ctx, r->fb_.get(), std::move(s), false));
            Adapter a;
            if (c.read_chunk_num == 1) a.base = std::move(pr);  // fs_reader_buffer.rs:181-183
            else a.chan.reset(new PrefetchChannel(std::move(pr), static_cast<size_t>(c.read_chunk_num)));
            r->readers_.push_back(std::move(a));
        }
    Adapter base;  // the random-read base reader
    base.base.reset(new FsReaderParallel(ctx, r->fb_.get(), {{0, r->len_}}, true));
    r->readers_.push_back(std::move(base));
    *out = std::move(r);
    return Err::ok();
}

Err FsReader::buffer_read() {
    chunk_off_ = 0;
    if (bpos_ >= len_) {
        chunk_.clear();
        return Err::ok();
    }
    const int64_t id = det_.is_random() ? det_.read_parallel : (bpos_ / slice_size_) % det_.read_parallel;
    if (id < 0 || id >= static_cast<int64_t>(readers_.size())) {
        chunk_.clear();
        return Err::common(str_printf("reader %lld is not initialized", (long long)id));
    }
    const double t0 = now_sec();
    int64_t off = 0;
    if (Err e = readers_[static_cast<size_t>(id)].read(&off, &chunk_)) {  // chunk_'s storage is handed down for reuse; nothing of it survives an error
        chunk_.clear();
        return e;
    }
    const int64_t diff = bpos_ - off;
    if (diff == 0) {
    } else if (diff > 0 && diff <= static_cast<int64_t>(chunk_.size())) {
        chunk_off_ = static_cast<size_t>(diff);  // misaligned first chunk: drop the excess prefix
    } else {
        chunk_.clear();
        return Err::common(str_printf("read data error: chunk offset %lld, pos %lld, diff %lld", (long long)off, (long long)bpos_, (long long)diff));
    }
    const int64_t n = static_cast<int64_t>(chunk_.size() - chunk_off_);
    const int64_t start = bpos_;
    bpos_ += n;
    if (det_.record_read(start, bpos_) && det_.is_sequential())
        for (auto& r : readers_) CV_RETURN_IF_ERR(r.pause(bpos_, false));  // fs_reader_buffer.rs:304-313
    ctx_->read_bytes += n;
    ctx_->read_time_us += static_cast<int64_t>((now_sec() - t0) * 1e6);
    return Err::ok();
}

Err FsReader::buffer_seek(int64_t pos) {
    if (pos == bpos_) return Err::ok();
    det_.record_seek();
    for (auto& r : readers_) {  // fs_reader_buffer.rs:325-337
        CV_RETURN_IF_ERR(r.seek(pos));
        if (!det_.enabled) CV_RETURN_IF_ERR(r.pause(pos, false));
    }
    bpos_ = pos;
    return Err::ok();
}

Err FsReader::read_chunk(const uint8_t** ptr, int64_t* n, int64_t max_len) {
    if (chunk_off_ >= chunk_.size()) CV_RETURN_IF_ERR(buffer_read());
    int64_t avail = static_cast<int64_t>(chunk_.size() - chunk_off_);
    if (max_len >= 0 && max_len < avail) avail = max_len;
    *ptr = reinterpret_cast<const uint8_t*>(chunk_.data()) + chunk_off_;
    *n = avail;
    chunk_off_ += static_cast<size_t>(avail);
    pos_ += avail;
    return Err::ok();
}

Err FsReader::read(uint8_t* buf, int64_t cap, int64_t* n) {
    const uint8_t* p;
    CV_RETURN_IF_ERR(read_chunk(&p, n, cap));
    if (*n > 0) memcpy(buf, p, static_cast<size_t>(*n));
    return Err::ok();
}

Err FsReader::read_full(uint8_t* buf, int64_t cap, int64_t* n) {
    int64_t off = 0;
    while (off < cap) {
        int64_t got = 0;
        CV_RETURN_IF_ERR(read(buf + off, cap - off, &got));
        if (got == 0) break;
        off += got;
    }
    *n = off;
    return Err::ok();
}

Err FsReader::seek(int64_t pos) {
    if (pos < 0) return Err::common("Cannot seek to negative offset");
    if (pos == pos_) return Err::ok();
    const int64_t skip = pos - pos_;
    const int64_t have = static_cast<int64_t>(chunk_.size() - chunk_off_);
    if (skip >= 0 && skip <= have) {
        chunk_off_ += static_cast<size_t>(skip);
    } else {
        chunk_.clear();
        chunk_off_ = 0;
        CV_RETURN_IF_ERR(buffer_seek(pos));
    }
    pos_ = pos;
    return Err::ok();
}

Err FsReader::complete() {
    Err first;
    for (auto& r : readers_) {
        Err e = r.complete();
        if (e && !first) first = e;
    }
    return first;
}

// ------------------------------------------------------------------ PrefetchChannel (fs_reader_buffer.rs:42-94,332-406)

PrefetchChannel::~PrefetchChannel() {
    {
        std::lock_guard<std::mutex> lk(mu_);
        if (started_ && !exited_) tasks_.push_back(Task{2, 0, false, 0});
        cv_.notify_all();
    }
    if (th_.joinable()) th_.join();
}

void PrefetchChannel::start_locked() {
    if (started_) return;
    started_ = true;
    th_ = std::thread([this] { loop(); });
}

// read_future: control messages first (biased select), then one chunk whenever the queue has room and the task is not paused
void PrefetchChannel::loop() {
    std::unique_lock<std::mutex> lk(mu_);
    for (;;) {
        if (!tasks_.empty()) {
            const Task t = tasks_.front();
            tasks_.pop_front();
            lk.unlock();
            Err e;
            if (t.kind == 0) e = reader_->seek(t.pos);
            else if (t.kind == 1) e = reader_->seek(t.pos);
            else e = reader_->complete();
            lk.lock();
            if (t.kind == 0) paused_ = true;
            if (t.kind == 1) paused_ = t.flag;
            if (t.ticket) done_ticket_ = std::max(done_ticket_, t.ticket);
            if (e && !err_) err_ = e;
            if (e || t.kind == 2) break;
            cv_.notify_all();
            continue;
        }
        if (!paused_ && q_.size() < cap_) {
            std::string buf;
            if (!spare_.empty()) {  // a chunk buffer the consumer is done with: same size as the next chunk, so no allocation and no zero fill
                buf = std::move(spare_.back());
                spare_.pop_back();
            }
            lk.unlock();
            int64_t off = 0;
            Err e = reader_->read(&off, &buf);
            lk.lock();
            if (e) {
                if (!err_) err_ = e;
                break;
            }
            if (buf.empty()) paused_ = true;  // out of slices: an empty chunk is sent so a reader never blocks, then wait for a command
            q_.emplace_back(off, std::move(buf));
            cv_.notify_all();
            continue;
        }
        cv_.wait(lk);
    }
    exited_ = true;
    cv_.notify_all();
}

Err PrefetchChannel::read(int64_t* off, std::string* buf) {
    std::unique_lock<std::mutex> lk(mu_);
    start_locked();
    cv_.wait(lk, [&] { return !q_.empty() || exited_; });
    if (q_.empty()) {
        buf->clear();
        return err_ ? err_ : Err::io("prefetch channel closed");
    }
    *off = q_.front().first;
    std::swap(*buf, q_.front().second);  // the consumer's previous chunk storage goes back to the producer
    if (q_.front().second.capacity() && spare_.size() < cap_) spare_.push_back(std::move(q_.front().second));
    q_.pop_front();
    cv_.notify_all();
    return Err::ok();
}

Err PrefetchChannel::seek(int64_t pos) {
    std::unique_lock<std::mutex> lk(mu_);
    start_locked();
    if (exited_) return err_ ? err_ : Err::io("prefetch channel closed");
    const uint64_t ticket = next_ticket_++;
    tasks_.push_back(Task{0, pos, false, ticket});
    cv_.notify_all();
    cv_.wait(lk, [&] { return done_ticket_ >= ticket || exited_; });
    if (done_ticket_ < ticket) return err_ ? err_ : Err::io("prefetch channel closed");
    q_.clear();  // everything prefetched before the seek is stale (the task is paused now: nothing new arrives)
    return err_;
}

Err PrefetchChannel::pause(int64_t pos, bool paused) {
    std::unique_lock<std::mutex> lk(mu_);
    start_locked();
    if (exited_) return err_ ? err_ : Err::io("prefetch channel closed");
    tasks_.push_back(Task{1, pos, paused, 0});
    cv_.notify_all();
    return Err::ok();
}

Err PrefetchChannel::complete() {
    std::unique_lock<std::mutex> lk(mu_);
    if (!started_) return reader_->complete();  // never used: nothing is open
    if (!exited_) {
        const uint64_t ticket = next_ticket_++;
        tasks_.push_back(Task{2, 0, false, ticket});
        cv_.notify_all();
        cv_.wait(lk, [&] { return exited_; });
    }
    lk.unlock();
    if (th_.joinable()) th_.join();
    return err_;
}

}  // namespace cv
