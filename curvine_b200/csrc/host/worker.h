// Worker-side read path: the per-connection ReadBlock handler over a BlockStore, served on TCP.
//
// Mirrors (reference):
//   orpc/src/server/rpc_server.rs:163-193, orpc/src/handler/stream_handler.rs:47-100   accept loop, per-connection
//        receive -> handle -> send; handler errors become error *responses* (block_handler.rs:57-60)
//   curvine-server/src/worker/handler/worker_handler.rs:42-98    one stateful BlockHandler per connection,
//        replaced on every non-Running message, dropped after Cancel/Complete
//   curvine-server/src/worker/handler/read_handler.rs:60-207     open / read / complete
//   curvine-server/src/worker/handler/context.rs:61-78           ReadContext::from_req
//   orpc/src/io/local_file.rs:103-117                            read_region: chunk = min(chunk_size, len - pos)
//   orpc/src/handler/rpc_frame.rs:97-121, orpc/src/sys/sys_libc.rs:76-122  payload by sendfile(2)
#pragma once
#include <atomic>
#include <memory>
#include <thread>

#include "block_store.h"
#include "hbm_tier.h"
#include "wire.h"

namespace cv {

struct WorkerMetrics {  // worker_metrics.rs:25-44
    std::atomic<int64_t> read_bytes{0}, read_time_us{0}, read_count{0}, read_blocks_local{0}, read_blocks_remote{0};
    std::atomic<int64_t> write_bytes{0}, write_time_us{0}, write_count{0}, write_blocks{0};
    std::atomic<int64_t> read_blocks_hbm{0}, hbm_packed_bytes{0};
};

// One request message as received from the socket.
struct RpcRequest {
    Protocol proto;
    std::string header;
    std::string data;
};

// What to send back: prefix(+header) and either inline data or a file region.
struct RpcResponse {
    Protocol proto;
    std::string header;
    std::string data;   // inline payload (errors, pread mode)
    const uint8_t* raw = nullptr;  // a ready-made wire image (prefix + payload, packed on the GPU): sent verbatim
    size_t raw_len = 0;
    int file_fd = -1;   // sendfile region when >= 0
    int64_t file_off = 0;
    int32_t file_len = 0;
    const uint8_t* mem = nullptr;  // payload straight out of the worker's mapping of a mem-arena segment (send(2), no page lookups)
    int32_t mem_len = 0;
    bool empty = false;
};

class ReadHandler {
   public:
    ReadHandler(BlockStore* store, WorkerMetrics* m, bool enable_send_file, HbmTier* hbm = nullptr)
        : store_(store), metrics_(m), enable_send_file_(enable_send_file), hbm_(hbm) {}
    ~ReadHandler();
    Err handle(const RpcRequest& req, RpcResponse* resp);

   private:
    Err open(const RpcRequest& req, RpcResponse* resp);
    Err read(const RpcRequest& req, RpcResponse* resp);
    Err complete(const RpcRequest& req, RpcResponse* resp);
    void read_ahead();
    BlockStore* store_;
    WorkerMetrics* metrics_;
    bool enable_send_file_;
    bool has_ctx_ = false;
    BlockReadRequest ctx_;
    int64_t ctx_req_id_ = 0;
    int fd_ = -1;
    int64_t pos_ = 0, len_ = 0, last_ahead_ = -1;
    bool is_tmpfs_ = false;
    std::string path_;
    BlockMeta meta_;  // an arena block's meta keeps its extent allocated for as long as this context lives
    // HBM tier: the whole response stream of this read, packed by K4 at Open
    HbmTier* hbm_ = nullptr;
    bool from_hbm_ = false;
    HbmBlock hbm_block_;
    PackedStream packed_;
    int32_t next_seq_ = 1;
};

// Write-side mirror (SURVEY.md 8f-1): WriteBlock = 80, Open{BlockWriteRequest} -> Running{payload, optional
// DataHeaderProto for seek/flush} x N -> Complete{BlockWriteRequest{block.len}} | Cancel
// (curvine-server/src/worker/handler/write_handler.rs:90-300).
class WriteHandler {
   public:
    WriteHandler(BlockStore* store, WorkerMetrics* m, HbmTier* hbm = nullptr) : store_(store), metrics_(m), hbm_(hbm) {}
    ~WriteHandler();
    Err handle(const RpcRequest& req, RpcResponse* resp);

   private:
    Err open(const RpcRequest& req, RpcResponse* resp);
    Err write(const RpcRequest& req, RpcResponse* resp);
    Err complete(const RpcRequest& req, RpcResponse* resp, bool commit);
    BlockStore* store_;
    WorkerMetrics* metrics_;
    HbmTier* hbm_ = nullptr;
    bool has_ctx_ = false, is_commit_ = false;
    BlockWriteRequest ctx_;
    int64_t ctx_req_id_ = 0;
    int fd_ = -1;
    int64_t pos_ = 0;
    BlockWriteTarget target_;  // the file or arena extent this context writes to
    bool target_open_ = false;
};

class Worker {
   public:
    Worker() = default;
    ~Worker();
    Err start(const std::vector<std::string>& data_dirs, const std::string& cluster_id, const std::string& host, int port, bool enable_send_file,
              const ArenaOpts& arena = ArenaOpts());
    void stop();
    int port() const { return port_; }
    BlockStore& store() { return store_; }
    HbmTier& hbm() { return hbm_; }
    WorkerMetrics& metrics() { return metrics_; }

   private:
    void accept_loop(int listen_fd);
    void serve(int fd);
    BlockStore store_;
    HbmTier hbm_;
    WorkerMetrics metrics_;
    int listen_fd_ = -1, unix_fd_ = -1;  // TCP, and the same-host abstract unix socket named after the TCP port (net.h)
    int wake_fd_ = -1;  // eventfd that stop() signals; the accept loops poll it beside their listening socket
    std::thread unix_accept_thread_;
    int port_ = 0;
    bool enable_send_file_ = true;
    std::atomic<bool> stopping_{false};
    std::thread accept_thread_;
    std::mutex conn_mu_;
    std::vector<int> conn_fds_;
    std::atomic<int> live_conns_{0};
};

}  // namespace cv
