// GPU ingest pipeline: blocks of a file -> HBM on side streams -> on-GPU CRC verify (-> page scatter).
//
// No reference counterpart (the reference has no GPU code); it replaces, for HBM destinations, the role of
// FsReaderBuffer's prefetch tasks (curvine-client/src/file/fs_reader_buffer.rs:332-406) and the caller's
// read_full + crc32 loop (curvine-tests/src/curvine_bench.rs:222-231), speaking the same worker protocol as
// BlockReaderLocal / BlockReaderRemote (block_reader_local.rs:43-143, block_reader_remote.rs:36-122):
//   arena          Open(short_circuit, accept_arena) names (segment, offset): DMA straight out of the arena segment this context
//                  pinned once at mount (arena.h) -> K1 CRC on the landed bytes; Complete sent without waiting for its answer
//   files          Open(short_circuit=true) -> block file: registered-mapping cache, or pread into a pinned slot -> H2D -> K1
//   disk tiers     cuFileRead file -> HBM (gds.h) where GPUDirect Storage is available; pinned ring otherwise
//   framed         Open + every Running request + Complete in one write -> the response stream (22-byte prefixes + payloads)
//                  received verbatim into a pinned slot -> H2D wire image -> K2 validates the prefixes, gathers payloads to
//                  their file offsets (clipping the tail of a ranged read) and CRCs them in the same pass
#pragma once
#include <atomic>
#include <condition_variable>
#include <thread>

#include "readv_plan.h"

namespace cv {

struct GpuReadStats {
    uint64_t bytes = 0;         // payload bytes landed in HBM
    uint64_t blocks = 0;        // block jobs
    uint64_t verified = 0;      // blocks whose CRC was compared with the manifest
    uint64_t h2d_bytes = 0;     // bytes moved by cudaMemcpyAsync (payload, + prefixes when framed)
    uint64_t kernel_launches = 0;
    uint64_t reg_hits = 0, reg_misses = 0;  // registered-mapping cache (zero-copy path), context-wide
    uint64_t reg_rejected = 0;              // mappings not admitted because the cache was full of in-use or recently used ones
    uint64_t reg_bytes = 0;                 // bytes registered through the cache right now (<= register_cache)
    double fetch_sec = 0;       // summed over fetch threads: time inside pread/recv
    double wall_sec = 0;
    uint64_t gds_bytes = 0;     // bytes that went file -> HBM through cuFileRead (gds.h)
    double ring_alloc_sec = 0;  // context-wide: one-off pinned-ring allocation time
};

class GpuIngest;  // per-FsContext pinned ring + streams
struct RegMapping;

class GpuFsReader {
   public:
    static Err open(FsContext* ctx, const std::string& path, std::unique_ptr<GpuFsReader>* out);
    ~GpuFsReader();
    int64_t len() const { return fbp_->status.len; }
    int64_t pos() const { return pos_; }
    Err seek(int64_t pos);
    const FileBlocks& file_blocks() const { return *fbp_; }
    // Next min(cap, remaining) bytes -> d_dst, ordered on `stream` when the call returns.  *n = bytes.
    Err read_device(void* d_dst, int64_t cap, void* stream, int64_t* n);
    // FUSE-shaped: the next min(len, remaining) bytes land in d_scratch and are scattered into page buffers
    // (d_page_base + page_offsets[i], page_size bytes each, the last one partial).
    Err fuse_read_device(int64_t len, void* d_scratch, void* d_page_base, const uint64_t* page_offsets, int64_t n_pages, int64_t page_size, void* stream,
                         int64_t* n);
    // Round-robin shard of the whole file: blocks b with b % world == rank land back to back in slots of
    // block_size bytes (slot j = block j*world + rank).  *n = bytes landed (sum of those block lengths).
    Err read_device_sharded(int rank, int world, void* d_dst, int64_t cap, void* stream, int64_t* n);
    // Vectored read (plan_readv): every touched block is fetched once and its CRC compared over the whole block.  Ordered on `stream`
    // when the call returns; does not move pos.  *n = bytes delivered: sum of rows * row_len (converted to destination bytes).
    Err readv_device(const ReadvRange* ranges, int32_t n_ranges, void* stream, int64_t* n);
    // Waits for outstanding work; sum_crc = u64 sum of the per-block CRCs computed so far (verify_poly),
    // n_bad = blocks whose CRC differed from the manifest.
    Err verify(uint64_t* sum_crc, uint32_t* n_bad, uint64_t* n_verified);
    const GpuReadStats& stats() const { return stats_; }
    Err complete();
    // Many whole files in one pipelined call (small-file batching, C5): file i lands at d_dst + dst_offs[i].
    // Blocks until verified.  Static: uses a throw-away reader on the context's ingest.
    static Err read_many(FsContext* ctx, const std::vector<std::string>& paths, const int64_t* dst_offs, void* d_dst, int64_t cap, void* stream,
                         uint64_t* sum_crc, uint32_t* n_bad, uint64_t* n_verified, int64_t* total_bytes);

   private:
    struct Job {
        const LocatedBlock* lb;  // the block (owned by a FileBlocks kept alive for the call)
        int64_t block_off;   // first byte of the block this job needs
        int64_t n;           // bytes
        int64_t dst_off;     // where they go in d_dst
        bool full;           // whole block -> CRC comparable with the manifest
    };
    // Layout of the per-call device tables (shared by all readers of the context) and of their pinned host image:
    //   off[J] len[J] expect[J] skip[J] | scatter section | crc[J] nbad[4] ferr[F] | streams[J] fdesc[F]
    // off .. the scatter section are uploaded in one copy before the fetch starts; crc .. ferr are the result words copied back.
    struct TableLayout {
        size_t J = 0, F = 0, o_len = 0, o_exp = 0, o_skip = 0, o_scatter = 0, o_crc = 0, o_streams = 0, o_fdesc = 0, bytes = 0;
        TableLayout() = default;
        TableLayout(size_t j, size_t f, size_t scatter_bytes);
        size_t res_words() const { return J + 4 + F; }
        uint64_t* off(uint8_t* t) const { return reinterpret_cast<uint64_t*>(t); }
        uint64_t* len(uint8_t* t) const { return reinterpret_cast<uint64_t*>(t + o_len); }
        uint32_t* expect(uint8_t* t) const { return reinterpret_cast<uint32_t*>(t + o_exp); }
        uint8_t* skip(uint8_t* t) const { return t + o_skip; }
        uint8_t* scatter(uint8_t* t) const { return t + o_scatter; }
        uint32_t* crc(uint8_t* t) const { return reinterpret_cast<uint32_t*>(t + o_crc); }
        // within the result words `res` (crc(t) in the tables, or the pinned mirror they are copied back to)
        uint32_t* nbad(uint32_t* res) const { return res + J; }      // mismatch counter (cvk_verify_crcs_masked)
        uint32_t* ferr(uint32_t* res) const { return res + J + 4; }  // frame flags (cvk_unpack_frames)
        CvStreamDesc* streams(uint8_t* t) const { return reinterpret_cast<CvStreamDesc*>(t + o_streams); }
        CvFrameDesc* fdesc(uint8_t* t) const { return reinterpret_cast<CvFrameDesc*>(t + o_fdesc); }
    };
    GpuFsReader() = default;
    struct Scatter;   // delivery riding on a read: spans of the landed bytes copied or converted to their destinations
    struct CallPlan;  // what one run_jobs call does, decided up front (plan_call)
    struct Call;      // one run_jobs call in flight: its tables, fetch workers, super-slot handoff, verifier and finish
    Err plan_call(const std::vector<Job>& jobs, size_t scatter_bytes, CallPlan* out) const;
    Err run_jobs(const std::vector<Job>& jobs, uint8_t* d_dst, void* stream, const Scatter* scatter = nullptr);
    Err read_device_impl(void* d_dst, int64_t cap, void* stream, int64_t* n, const Scatter* scatter);
    FsContext* ctx_ = nullptr;
    std::shared_ptr<const FileBlocks> fbp_;
    int64_t pos_ = 0;
    GpuReadStats stats_;
    GpuIngest* ing_ = nullptr;
    uint64_t sum_crc_ = 0, n_verified_ = 0;
    uint32_t n_bad_ = 0;
    uint64_t n_bad_frames_ = 0;
    uint32_t first_frame_err_ = 0;
    std::vector<std::shared_ptr<struct RegMapping>> held_maps_;  // registered mappings with copies still in flight (until harvest)
    std::vector<std::shared_ptr<const FileBlocks>> held_files_;  // read_many: keeps the LocatedBlocks alive
    struct Pending {
        bool active = false;
        TableLayout tl;  // of the call whose result words sit in h_result
        size_t f0 = 0, f1 = 0, n_compared = 0;
    } pending_;
    Err harvest();
    friend class GpuIngest;
};

// one per (process, device): pinned ring, device staging ring, streams, events
GpuIngest* gpu_ingest_get(FsContext* ctx, Err* err);
void gpu_ingest_release(FsContext* ctx);
void gpu_ingest_wait_registered(FsContext* ctx);  // block until the background registrar is idle and every queued arena segment is pinned
Err gpu_ingest_preregister(FsContext* ctx);       // create the context's ingest now: `arena_preregister` dirs start being pinned
void gpu_ingest_arena_stats(FsContext* ctx, uint64_t out[5]);

}  // namespace cv
