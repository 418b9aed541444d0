// orpc RpcMessage frame codec + the protobuf headers on the block-read path.
//
// Mirrors (reference, relative to the CurvineIO/curvine source tree):
//   orpc/src/message/rpc_message.rs:26-41,43-90,301-338   Protocol / Status / encode_protocol / decode_protocol
//   orpc/src/handler/rpc_frame.rs:205-264                  Frame::send / Frame::receive (heartbeats skipped)
//   orpc/src/error/error_encoder.rs:24-51                  error body layout
//   curvine-common/proto/worker.proto:38-60                BlockReadRequest / BlockReadResponse / DataHeaderProto
//   curvine-common/src/fs/rpc_code.rs:76-79                ReadBlock = 81
#pragma once
#include <vector>

#include "common.h"

namespace cv {

constexpr int32_t kProtocolSize = 22;
constexpr int32_t kHeadSize = 18;
constexpr int32_t kMaxDataSize = 16 * 1024 * 1024;

constexpr int8_t kCodeWriteBlock = 80;
constexpr int8_t kCodeReadBlock = 81;

enum RequestStatus : int8_t { kReqUndefined = -1, kReqHeartbeat = 0, kReqRpc = 1, kReqOpen = 2, kReqRunning = 3, kReqCancel = 4, kReqComplete = 5 };
enum ResponseStatus : int8_t { kRespUndefined = -1, kRespSuccess = 0, kRespError = 1 };

// StorageTypeProto (common.proto:9-16)
enum StorageType : int32_t { kStorageMem = 0, kStorageSsd = 1, kStorageHdd = 2, kStorageUfs = 3, kStorageDisk = 4, kStorageSpdkDisk = 5 };

inline int8_t status_encode(int8_t req, int8_t resp) {
    return static_cast<int8_t>(static_cast<uint8_t>(req) | static_cast<uint8_t>(static_cast<uint8_t>(resp) << 4));
}
inline void status_decode(int8_t v, int8_t* req, int8_t* resp) {
    int8_t r = v & 0x0f, s = static_cast<int8_t>(v >> 4);
    *req = (r >= 0 && r <= 5) ? r : kReqUndefined;
    *resp = (s == 0 || s == 1) ? s : kRespUndefined;
}

struct Protocol {
    int8_t code = 0;
    int8_t req_status = kReqUndefined;
    int8_t resp_status = kRespUndefined;
    int64_t req_id = 0;
    int32_t seq_id = 0;
    int32_t header_len = 0;
    int32_t data_len = 0;
    bool is_success() const { return resp_status == kRespSuccess; }
    bool is_heartbeat() const { return req_status == kReqHeartbeat; }
};

// writes the 22-byte prefix
void encode_protocol(const Protocol& p, uint8_t out[kProtocolSize]);
// rpc_message.rs:326-338: rejects data_len < 0 and > 16 MiB
Err decode_protocol(const uint8_t in[kProtocolSize], Protocol* p);
// a request's prefix fields; header_len and data_len are set where the frame is encoded
Protocol request_proto(int8_t code, int8_t req_status, int64_t req_id, int32_t seq_id);

struct BlockReadRequest {  // worker.proto:38-47
    int64_t id = 0, off = 0, len = 0;
    int32_t chunk_size = 0;
    bool short_circuit = false;
    bool enable_read_ahead = true;
    int64_t read_ahead_len = 4194304;
    int64_t drop_cache_len = 1048576;
    // extension (optional field 100, skipped as unknown by a prost/proto2 decoder): the client understands arena
    // extents, i.e. a short-circuit response whose `path` is an arena segment plus `arena_off` (arena.h)
    bool accept_arena = false;
    std::string encode() const;
    static Err decode(const uint8_t* p, size_t n, BlockReadRequest* out);
};

struct BlockReadResponse {  // worker.proto:49-54
    int64_t id = 0, len = 0;
    bool has_path = false;
    std::string path;
    int32_t storage_type = kStorageDisk;
    // extension (optional fields 100/101, only sent to a client that said accept_arena): the block is bytes
    // [arena_off, arena_off + len) of the segment file `path`, which is arena_seg_len bytes long
    bool has_arena = false;
    int64_t arena_off = 0, arena_seg_len = 0;
    std::string encode() const;
    static Err decode(const uint8_t* p, size_t n, BlockReadResponse* out);
};

struct DataHeaderProto {  // worker.proto:56-60
    int64_t offset = 0;
    bool flush = false, is_last = false;
    std::string encode() const;
    static Err decode(const uint8_t* p, size_t n, DataHeaderProto* out);
};

struct ExtendedBlockWire {  // common.proto:98-104 (ExtendedBlockProto); block_size carries the block's current length
    int64_t id = 0, block_size = 0;
    int32_t storage_type = kStorageDisk, file_type = 1;  // FILE_TYPE_PROTO_FILE
};

struct BlockWriteRequest {  // worker.proto:10-18
    ExtendedBlockWire block;
    int64_t off = 0, block_size = 0;
    bool short_circuit = false;
    std::string client_name;
    int32_t chunk_size = 0;
    std::string encode() const;
    static Err decode(const uint8_t* p, size_t n, BlockWriteRequest* out);
};

struct BlockWriteResponse {  // worker.proto:27-34
    int64_t id = 0;
    bool has_path = false;
    std::string path;
    int64_t off = 0, block_size = 0;
    int32_t storage_type = kStorageDisk;
    std::string encode() const;
    static Err decode(const uint8_t* p, size_t n, BlockWriteResponse* out);
};

std::string encode_error_body(int32_t kind, const std::string& msg);
Err decode_error_body(const uint8_t* p, size_t n);  // always returns a failure Err carrying kind + message

// Folded UUID-ish request id (orpc/src/common/utils.rs:35-41): any i64 works on the wire.
int64_t new_req_id();

}  // namespace cv
