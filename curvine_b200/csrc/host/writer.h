// Write-side mirror of the block path (SURVEY.md 8f-1): client block writer + its CUDA counterpart.
//
// Mirrors (reference):
//   curvine-client/src/block/block_client.rs:97-219      write_block / write_data / write_flush / write_commit
//   curvine-client/src/block/block_writer_remote.rs:36-140  Open (seq 0) -> Running x N (seq 1..) -> Complete (seq n+1)
//   curvine-client/src/file/fs_writer_base.rs             a file = blocks of block_size allocated one after another
// Master-side add_block / complete_file are out of scope: block ids are inode<<24|seq (inode_id.rs:48-60) and the
// finished file is registered in the context's namespace with the per-block CRCs computed AT WRITE TIME
// (the write-sum == read-sum discipline of worker_test.rs:54-57 / block_test.rs:209-226).
// Device path: the payload already lives in HBM; K4 (cvk_pack_frames) writes the Running-request prefixes and copies
// the payload behind them while CRC-ing the source, the wire image goes D2H once and onto the socket verbatim.
#pragma once
#include "client.h"
#include "packed_frames.h"

namespace cv {

class FsWriter {
   public:
    static Err create(FsContext* ctx, const std::string& path, int64_t inode_id, int64_t block_size, int32_t storage_type,
                      const WorkerAddress& worker, int64_t chunk_size, std::unique_ptr<FsWriter>* out);
    ~FsWriter();
    Err write(const uint8_t* buf, int64_t n);                  // host bytes
    Err write_device(const void* d_src, int64_t n, void* stream);  // HBM bytes (K4 pack + CRC at source)
    Err complete();                                            // commit the open block, register the file
    Err cancel();
    int64_t pos() const { return pos_; }
    std::string manifest() const;

   private:
    FsWriter() = default;
    Err open_block();
    Err commit_block(bool cancel);
    Err send_running(const uint8_t* payload, int64_t n);
    FsContext* ctx_ = nullptr;
    FileBlocks fb_;
    WorkerAddress worker_;
    int64_t block_size_ = 0, chunk_size_ = 0, pos_ = 0;
    int32_t storage_type_ = kStorageDisk;
    std::unique_ptr<BlockClient> client_;
    bool block_open_ = false;
    int64_t block_pos_ = 0, req_id_ = 0;
    int32_t seq_ = 0;
    uint32_t crc32_ = 0, crc32c_ = 0;  // running CRCs of the open block
    PackedStream packed_;  // write_device's wire image, reused from call to call
    bool done_ = false;
};

uint32_t host_crc_update(int poly, uint32_t crc, const uint8_t* buf, size_t len);

}  // namespace cv
