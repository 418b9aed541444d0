// Client reader stack (host side): namespace lookup, block RPC client + pool, block readers with replica
// failover, and the file-level reader that implements the reference `Reader` trait semantics.
//
// Mirrors (reference, relative to the CurvineIO/curvine source tree):
//   curvine-common/src/state/block_info.rs:66-72,127-131,156-217   ExtendedBlock / LocatedBlock / FileBlocks / search
//   curvine-client/src/block/block_client.rs:222-300               open_block / read_data / read_commit
//   orpc/src/client/raw_client.rs:100-116                          req_id/seq_id echo check
//   curvine-client/src/block/block_client_pool.rs:90-168           LIFO idle pool per worker
//   curvine-client/src/block/block_reader.rs:116-254               replica choice + failover
//   curvine-client/src/block/block_reader_{remote,local,hole}.rs   the three adapters
//   curvine-client/src/file/fs_reader_base.rs:101-204              block cursor + parked-reader cache
//   curvine-client/src/file/fs_reader_parallel.rs:94-187           slice striping
//   curvine-client/src/file/fs_reader_buffer.rs:248-323            sub-reader choice, misaligned trim
//   curvine-client/src/file/read_detector.rs:130-218               sequential/random detector
//   curvine-client/src/file/fs_reader.rs:103-126                   seek fast path
//   curvine-common/src/fs/reader.rs:50-141                         read_chunk / read / read_full / fuse_read
//   curvine-client/src/file/fs_reader_buffer.rs:30-94,147-222,332-406  prefetch tasks: one per striped sub-reader, a
//        bounded channel of read_chunk_num chunks each, Seek / Pause / Stop control messages (PrefetchChannel below)
#pragma once
#include <atomic>
#include <condition_variable>
#include <deque>
#include <list>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <vector>

#include "conf.h"
#include "wire.h"

namespace cv {

struct WorkerAddress {
    uint32_t worker_id = 0;
    std::string hostname, ip_addr;
    uint32_t rpc_port = 0, web_port = 0;
    bool operator==(const WorkerAddress& o) const { return hostname == o.hostname && rpc_port == o.rpc_port && worker_id == o.worker_id; }
    std::string str() const { return hostname + ":" + std::to_string(rpc_port); }
};

struct ExtendedBlock {
    int64_t id = 0, len = 0;
    int32_t storage_type = kStorageDisk;
    bool has_alloc_opts = false;  // block allocated but never written -> hole when it has no locations
};

struct LocatedBlock {
    ExtendedBlock block;
    std::vector<WorkerAddress> locs;
    uint32_t crc32 = 0, crc32c = 0;  // manifest: expected per-block CRCs (SURVEY.md §0 "what verify compares against")
    bool has_crc = false;
};

struct FileStatus {
    int64_t id = 0;
    std::string path;
    int64_t len = 0;
    int64_t block_size = 0;
    int64_t mtime = 0;
};

struct FileBlocks {
    FileStatus status;
    std::vector<LocatedBlock> block_locs;
    std::vector<int64_t> starts;  // prefix offsets (SearchFileBlocks::search_off)
    void build_index();
    // (block_off, index); partition_point(|x| x.end <= pos); error past the end
    Err get_read_block(int64_t pos, int64_t* block_off, size_t* index) const;
};

// file -> blocks table.  Stands in for master GetBlockLocations (master_handler.rs:409-418), which is out of scope.
class Namespace {
   public:
    Err load(const std::string& manifest_path);
    Err load_string(const std::string& text);
    Err get_block_locations(const std::string& path, std::shared_ptr<const FileBlocks>* out) const;  // shared, immutable
    void put(const FileBlocks& fb);
    std::string dump() const;

   private:
    mutable std::mutex mu_;
    std::map<std::string, std::shared_ptr<const FileBlocks>> files_;
};

// ------------------------------------------------------------------ block RPC client

// Every answer is read by recv_answer, and one rule decides whether the connection can still be used: any failure to send a request or
// to receive, frame or match (request and seq id) its answer marks it `broken`, and FsContext::release closes it instead of pooling it.  A
// well-formed error answer leaves it in step: the call returns the worker's error and the connection stays usable.  A call that has
// already sent more requests behind the failed one (open_blocks, send_block_read_pipeline, FsWriter::write_device) marks it broken on
// any error, since those answers may still be on the wire.
class BlockClient {
   public:
    BlockClient(int fd, WorkerAddress addr) : fd_(fd), addr_(std::move(addr)) {}
    ~BlockClient();
    int fd() const { return fd_; }
    const WorkerAddress& addr() const { return addr_; }
    // send one request frame and read its answer
    Err rpc(const Protocol& req, const std::string& header, Protocol* resp, std::string* resp_header, std::string* resp_data);
    // the answer to `req`: prefix and header (heartbeats skipped), the payload into *data (resized in place), the echo check, and an
    // error status decoded into the worker's Err
    Err recv_answer(const Protocol& req, Protocol* resp, std::string* header, std::string* data);
    // request frame -> the end of `out`: prefix + header; the caller sends the data_len payload bytes behind it
    static void append_frame(const Protocol& req, const std::string& header, std::string* out, int32_t data_len = 0);
    Err open_block(const ClientConf& conf, const ExtendedBlock& b, int64_t off, int64_t len, int64_t req_id, int32_t seq_id, bool short_circuit,
                   int64_t chunk_size, BlockReadResponse* out, bool accept_arena = false);
    Err read_commit(const ExtendedBlock& b, int64_t req_id, int32_t seq_id);
    // Complete without waiting for the answer (GPU reader: one round trip less per block).  The response is consumed -- and its
    // echo / status checked -- before the next request goes out on this connection (drain_pending), also after a trip through the pool.
    Err read_commit_deferred(const ExtendedBlock& b, int64_t req_id, int32_t seq_id);
    // Short-circuit Opens of several blocks in ONE write, then their answers in order (after those of the deferred Completes still
    // owed); Completes (seq_id 1) of several blocks in one write, deferred.  Same messages and request ids as one call per block.
    struct OpenReq {
        const ExtendedBlock* b;
        int64_t off, req_id;
    };
    Err open_blocks(const ClientConf& conf, const std::vector<OpenReq>& reqs, int64_t chunk_size, bool accept_arena, std::vector<BlockReadResponse>* out);
    Err read_commit_deferred(const std::vector<OpenReq>& reqs);
    Err drain_pending();
    size_t pending() const { return pending_.size(); }
    // Whole-block pipelining for the GPU reader's framed path: Open, every Running request and the Complete of one block leave in
    // ONE write (the worker serves a connection's requests in order); the Open answer is read first, then the caller receives the
    // data frames, and the Complete's answer stays pending like a deferred Complete.  Same messages, same order, two round trips less.
    Err send_block_read_pipeline(const ClientConf& conf, const ExtendedBlock& b, int64_t off, int64_t req_id, int64_t chunk_size, int64_t n_running,
                                 BlockReadResponse* open_resp);
    bool broken = false;
    int64_t idle_since_ms = 0;  // set when the connection goes back to the pool (BlockClient::uptime, block_client.rs:47,80-86)

   private:
    Err send_request(const Protocol& req, const std::string& header);
    int fd_;
    WorkerAddress addr_;
    std::vector<Protocol> pending_;  // requests whose responses are still on the wire (deferred Completes)
};

class FsContext {
   public:
    explicit FsContext(const ClusterConf& conf) : conf(conf) {}
    ~FsContext();
    ClusterConf conf;
    Namespace ns;
    // block_client_pool.rs:102-160: LIFO idle connections per worker; at most block_conn_idle_size idle connections over all
    // workers (a connection returned to a full pool is closed); a pooled connection idle for block_conn_idle_time or longer
    // is dropped when acquire meets it
    Err acquire_read(const WorkerAddress& addr, std::unique_ptr<BlockClient>* out);
    void release(std::unique_ptr<BlockClient> c);
    // keeps *conn when it goes to `addr` and is not broken; otherwise releases it and acquires a connection to `addr`
    Err connection_to(const WorkerAddress& addr, std::unique_ptr<BlockClient>* conn);
    bool is_local_worker(const WorkerAddress& addr) const { return addr.hostname == conf.client.hostname; }
    int64_t read_chunk_size() const { return conf.client.read_chunk_size; }
    // fs_context.rs:83-86,182-205: workers excluded for failed_worker_ttl.  As in the reference only the write path adds to the list;
    // the read path reports it in its "There is no available worker" error.
    void add_failed_worker(const WorkerAddress& addr);
    bool is_failed_worker(const WorkerAddress& addr);
    std::vector<uint32_t> get_failed_workers();
    // "There is no available worker, locs: [...], failed workers: [...]" (block_reader.rs:209-213)
    Err no_available_worker(const std::vector<WorkerAddress>& locs);
    // client metrics (client_metrics.rs:24-35)
    std::atomic<int64_t> read_bytes{0}, read_time_us{0};

   private:
    std::mutex mu_;
    std::unordered_map<std::string, std::vector<std::unique_ptr<BlockClient>>> idle_;
    int64_t idle_total_ = 0;  // cur_idle_size
    int64_t conns_opened_ = 0, conns_expired_ = 0;
    std::mutex fw_mu_;
    std::unordered_map<uint32_t, int64_t> failed_workers_;  // worker_id -> expiry (ms)
   public:
    void pool_stats(int64_t out[3]);  // idle now (BlockClientPool::idle_conn), connections opened so far, pooled connections dropped as expired
};

// ------------------------------------------------------------------ block readers

class BlockReader {
   public:
    // BlockReader::new: sort replicas (local first when short_circuit), open the first that works
    static Err create(FsContext* ctx, const LocatedBlock& lb, int64_t off, std::unique_ptr<BlockReader>* out);
    ~BlockReader();
    // next chunk: min(chunk_size, len - pos) bytes into *buf (resized); empty at end of block
    Err read(std::string* buf);
    Err seek(int64_t pos);
    Err complete();
    int64_t pos() const { return pos_; }
    int64_t len() const { return block_.len; }
    int64_t remaining() const { return block_.len - pos_; }
    bool has_remaining() const { return remaining() > 0; }
    int64_t block_id() const { return block_.id; }
    enum Kind { kLocal, kRemote, kHole };
    Kind kind() const { return kind_; }

   private:
    BlockReader() = default;
    Err open_adapter(int64_t off);
    Err read_once(std::string* buf);
    void drop_adapter();
    FsContext* ctx_ = nullptr;
    ExtendedBlock block_;
    std::vector<WorkerAddress> locs_;
    WorkerAddress cur_addr_;
    Kind kind_ = kHole;
    int64_t pos_ = 0;
    int64_t chunk_size_ = 0;
    // remote
    std::unique_ptr<BlockClient> client_;
    int64_t req_id_ = 0;
    int32_t seq_id_ = 0;
    bool pending_seek_ = false;
    // local
    int fd_ = -1;
    int64_t base_off_ = 0;  // where the block starts inside fd_ (non-zero for a mem-arena extent)
    bool ra_enabled_ = false;
    int64_t last_ahead_ = -1;
};

// ------------------------------------------------------------------ file-level reader

std::vector<std::vector<std::pair<int64_t, int64_t>>> split_slices(int64_t total, int64_t slice_size, int64_t read_parallel);

class ReadDetector {
   public:
    ReadDetector() = default;
    ReadDetector(const ClientConf& conf, int64_t file_size);
    bool enabled = true;
    int64_t read_parallel = 1;
    bool is_random() const { return random_; }
    bool is_sequential() const { return !random_; }
    uint64_t seq_count() const { return seq_count_; }
    void record_seek();
    bool record_read(int64_t start, int64_t end);
    void set_last_read_pos(int64_t p) { last_read_pos_ = p; }

   private:
    int64_t last_read_pos_ = -1;
    uint64_t seq_count_ = 0, threshold_ = 7;
    bool random_ = false;
};

class FsReaderBase {
   public:
    FsReaderBase(FsContext* ctx, const FileBlocks* fb, bool cache_handles);
    ~FsReaderBase();
    Err read(std::string* buf);  // empty at EOF
    Err seek(int64_t pos);
    Err complete();
    int64_t pos() const { return pos_; }

   private:
    Err update_reader(std::unique_ptr<BlockReader> cur, bool cache);
    Err get_reader();
    FsContext* ctx_;
    const FileBlocks* fb_;
    int64_t pos_ = 0, len_ = 0;
    std::unique_ptr<BlockReader> cur_;
    size_t cache_limit_;
    std::list<std::unique_ptr<BlockReader>> cache_;  // FIFO of parked (still open) readers
};

class FsReaderParallel {
   public:
    FsReaderParallel(FsContext* ctx, const FileBlocks* fb, std::vector<std::pair<int64_t, int64_t>> slices, bool cache_handles)
        : inner_(ctx, fb, cache_handles), slices_(std::move(slices)) {}
    Err read(int64_t* off, std::string* buf);
    Err seek(int64_t pos);
    Err complete() { return inner_.complete(); }

   private:
    FsReaderBase inner_;
    std::vector<std::pair<int64_t, int64_t>> slices_;
    int64_t cur_ = -1;
};

// BufferChannel + FsReaderBuffer::read_future (fs_reader_buffer.rs:42-94,332-406): a striped sub-reader owned by a prefetch
// thread that keeps up to `cap` chunks ahead of the consumer in a bounded queue.  Control messages as in the reference:
//   seek(pos)   the thread seeks its reader and PAUSES; the consumer then drops everything that was prefetched
//   pause(pos, paused)  seek + set the paused flag (resume = pause(pos, false)); fire and forget
//   stop()      complete() on the reader, thread exits
// An empty chunk (the sub-reader ran out of slices) is delivered too and pauses the thread; the first error ends the thread
// and is what every later read() returns.  The thread starts with the first use (the reference spawns its tasks in
// FsReaderBuffer::new; here a reader that is only ever used for device reads must not prefetch into host memory).
class PrefetchChannel {
   public:
    PrefetchChannel(std::unique_ptr<FsReaderParallel> reader, size_t cap) : reader_(std::move(reader)), cap_(std::max<size_t>(cap, 1)) {}
    ~PrefetchChannel();
    Err read(int64_t* off, std::string* buf);
    Err seek(int64_t pos);
    Err pause(int64_t pos, bool paused);
    Err complete();

   private:
    struct Task {
        int kind;  // 0 seek, 1 pause, 2 stop
        int64_t pos;
        bool flag;
        uint64_t ticket;
    };
    void start_locked();
    void loop();
    std::unique_ptr<FsReaderParallel> reader_;
    size_t cap_;
    std::thread th_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<std::pair<int64_t, std::string>> q_;
    std::vector<std::string> spare_;  // chunk buffers handed back by the consumer
    std::deque<Task> tasks_;
    uint64_t next_ticket_ = 1, done_ticket_ = 0;
    bool started_ = false, paused_ = false, exited_ = false;
    Err err_;
};

// FsReader + FsReaderBuffer + the provided methods of `trait Reader`
class FsReader {
   public:
    static Err open(FsContext* ctx, const std::string& path, std::unique_ptr<FsReader>* out);
    int64_t len() const { return len_; }
    int64_t pos() const { return pos_; }
    int64_t chunk_size() const { return chunk_size_; }
    const FileBlocks& file_blocks() const { return *fb_; }
    FsContext* ctx() const { return ctx_; }
    // Reader::read_chunk(None) + pos advance == blocking_read: borrowed pointer valid until the next call
    Err read_chunk(const uint8_t** ptr, int64_t* n, int64_t max_len = -1);
    Err read(uint8_t* buf, int64_t cap, int64_t* n);       // Reader::read
    Err read_full(uint8_t* buf, int64_t cap, int64_t* n);  // Reader::read_full
    Err seek(int64_t pos);
    Err complete();
    const ReadDetector& detector() const { return det_; }

   private:
    FsReader() = default;
    Err buffer_read();
    Err buffer_seek(int64_t pos);
    FsContext* ctx_ = nullptr;
    std::shared_ptr<const FileBlocks> fb_;
    int64_t len_ = 0, pos_ = 0, bpos_ = 0, chunk_size_ = 0, slice_size_ = 0;
    ReadDetector det_;
    // ReaderAdapter (fs_reader_buffer.rs:96-132): Buffer(channel) for the striped sub-readers when read_chunk_num > 1, Base otherwise
    struct Adapter {
        std::unique_ptr<PrefetchChannel> chan;
        std::unique_ptr<FsReaderParallel> base;
        Err read(int64_t* off, std::string* buf) { return chan ? chan->read(off, buf) : base->read(off, buf); }
        Err seek(int64_t pos) { return chan ? chan->seek(pos) : base->seek(pos); }
        Err pause(int64_t pos, bool paused) { return chan ? chan->pause(pos, paused) : base->seek(pos); }
        Err complete() { return chan ? chan->complete() : base->complete(); }
    };
    std::vector<Adapter> readers_;
    std::string chunk_;     // current chunk storage
    size_t chunk_off_ = 0;  // consumed prefix
    std::string tmp_;
};

}  // namespace cv
