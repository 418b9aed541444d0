#include "gpu_reader.h"

#include <cuda_runtime.h>
#include <errno.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <array>

#include "../../../include/curvine_b200_kernels.h"
#include "block_store.h"
#include "gds.h"
#include "net.h"
#include "numa.h"
#include "reg_cache.h"

namespace cv {

// ------------------------------------------------------------------ GpuIngest: ring + streams

class GpuIngest {
   public:
    int device = 0;
    int nslots = 0;
    size_t slot_bytes = 0;
    uint8_t* pinned = nullptr;
    uint8_t* d_stage = nullptr;  // framed mode only
    size_t d_stage_bytes = 0;
    std::vector<cudaEvent_t> copy_ev, free_ev;
    std::vector<cudaStream_t> copy_streams;
    cudaStream_t vstream = nullptr;
    cudaEvent_t done_ev = nullptr;
    std::vector<int> cpus;
    std::mutex mu;  // one read_device at a time per context
    // per-call device tables + pinned result mirror, shared by every reader of the context
    uint8_t* d_tables = nullptr;
    size_t d_tables_cap = 0;
    uint8_t* h_result = nullptr;
    size_t h_result_cap = 0;
    uint8_t* h_tables = nullptr;  // pinned image of the per-call tables (off/len/expect/skip, stream descriptors): uploads are truly
    size_t h_tables_cap = 0;      // asynchronous, nothing waits for them (a pageable source makes cudaMemcpyAsync drain the stream first)
    GpuFsReader* pending_owner = nullptr;  // reader whose results still sit in h_result
    RegCache reg;
    Registrar registrar;
    ArenaSegs arena;
    cudaEvent_t entry_ev = nullptr;  // what the caller's stream had queued when a read started
    bool register_inline = false;
    std::atomic<int> reads_in_flight{0};  // run_jobs calls between entry and return (the registrar yields to them)
    double ring_alloc_sec = 0;            // time spent allocating the pinned ring (one-off per context and slot size)
    // device staging of the boundary blocks of vectored reads (readv_device): one vectored read at a time uses it, under readv_mu
    std::mutex readv_mu;
    uint8_t* d_readv_stage = nullptr;
    size_t d_readv_stage_bytes = 0;

    Err ensure_readv_stage(size_t bytes) {
        if (bytes <= d_readv_stage_bytes) return Err::ok();
        CU_TRY(cudaDeviceSynchronize());  // an earlier vectored read's K3 may still be reading the old staging
        if (d_readv_stage) cudaFree(d_readv_stage);
        d_readv_stage = nullptr, d_readv_stage_bytes = 0;
        CU_TRY(cudaMalloc(&d_readv_stage, bytes));
        d_readv_stage_bytes = bytes;
        return Err::ok();
    }

    Err ensure_tables(size_t tables_bytes, size_t result_bytes) {
        if (tables_bytes > d_tables_cap) {
            if (d_tables) cudaFree(d_tables);
            d_tables_cap = tables_bytes * 2;
            CU_TRY(cudaMalloc(&d_tables, d_tables_cap));
        }
        if (tables_bytes > h_tables_cap) {
            if (h_tables) cudaFreeHost(h_tables);
            h_tables_cap = tables_bytes * 2;
            CU_TRY(cudaHostAlloc(&h_tables, h_tables_cap, cudaHostAllocDefault));
        }
        if (result_bytes > h_result_cap) {
            if (h_result) cudaFreeHost(h_result);
            h_result_cap = result_bytes * 2;
            CU_TRY(cudaHostAlloc(&h_result, h_result_cap, cudaHostAllocDefault));
        }
        return Err::ok();
    }

    Err init(const B200Conf& c) {
        device = c.device;
        CU_TRY(cudaSetDevice(device));
        CVK_TRY(cvk_init(device));
        const int kk = std::max(1, c.copy_group);
        nslots = std::max(c.pinned_slots, (2 * ((c.verify_batch + kk - 1) / kk) + c.fetch_threads + 2) * kk);
        nslots = (nslots + kk - 1) / kk * kk;
        copy_ev.resize(nslots), free_ev.resize(nslots);
        for (int i = 0; i < nslots; i++) {
            CU_TRY(cudaEventCreateWithFlags(&copy_ev[i], cudaEventDisableTiming));
            CU_TRY(cudaEventCreateWithFlags(&free_ev[i], cudaEventDisableTiming));
        }
        copy_streams.resize(static_cast<size_t>(std::max(1, std::min(c.copy_streams, c.fetch_threads))));
        for (auto& s : copy_streams) CU_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
        CU_TRY(cudaStreamCreateWithFlags(&vstream, cudaStreamNonBlocking));
        CU_TRY(cudaEventCreateWithFlags(&done_ev, cudaEventDisableTiming));
        CU_TRY(cudaEventCreateWithFlags(&entry_ev, cudaEventDisableTiming));
        reg.capacity = c.zero_copy ? static_cast<size_t>(std::max<int64_t>(c.register_cache, 0)) : 0;
        reg.min_age_sec = static_cast<double>(std::max<int64_t>(c.register_min_age_ms, 0)) / 1000.0;
        register_inline = c.register_threads <= 0 || reg.capacity == 0;
        // CPUs of the GPU's NUMA node: pinned pages and fetch threads stay next to the PCIe root
        int node = c.numa_node;  // -1: the GPU's node (auto); -2: do not bind the fetch threads
        if (node == -1) node = gpu_numa_node(device);
        cpus = node_cpus(node);
        if (c.zero_copy && !register_inline) registrar.start(c.register_threads, device, &reg, cpus, c.register_when_idle ? &reads_in_flight : nullptr);
        if (c.zero_copy && c.arena) arena.start(std::max(1, c.register_threads), device, cpus, static_cast<size_t>(std::max<int64_t>(c.arena_register_slice, 0)));
        else arena.unsupported.store(true);
        return Err::ok();
    }

    Err ensure(size_t need_slot_bytes, bool framed) {
        need_slot_bytes = page_up(need_slot_bytes);
        if (need_slot_bytes > slot_bytes) {
            CU_TRY(cudaDeviceSynchronize());
            if (pinned) cudaFreeHost(pinned);
            if (d_stage) cudaFree(d_stage);
            pinned = nullptr, d_stage = nullptr, d_stage_bytes = 0;
            slot_bytes = need_slot_bytes;
            // allocate the ring from a thread bound to the GPU's node (the driver allocates and pins the pages in that
            // thread's context, so they land on its node; no extra first-touch pass)
            Err err;
            const double t0 = now_sec();
            std::thread t([&] {
                bind_cpus(cpus);
                cudaSetDevice(device);
                cudaError_t e = cudaHostAlloc(&pinned, slot_bytes * nslots, cudaHostAllocDefault);
                if (e != cudaSuccess) err = Err::io(str_printf("cudaHostAlloc(%zu): %s", slot_bytes * nslots, cudaGetErrorString(e)));
            });
            t.join();
            ring_alloc_sec += now_sec() - t0;
            if (err) return err;
        }
        if (framed && d_stage_bytes < slot_bytes * nslots) {
            if (d_stage) cudaFree(d_stage);
            d_stage_bytes = slot_bytes * nslots;
            CU_TRY(cudaMalloc(&d_stage, d_stage_bytes));
        }
        return Err::ok();
    }

    ~GpuIngest() {
        registrar.stop();
        cudaSetDevice(device);
        cudaDeviceSynchronize();
        arena.stop();
        reg.clear();
        if (pinned) cudaFreeHost(pinned);
        if (d_stage) cudaFree(d_stage);
        if (d_readv_stage) cudaFree(d_readv_stage);
        if (d_tables) cudaFree(d_tables);
        if (h_result) cudaFreeHost(h_result);
        if (h_tables) cudaFreeHost(h_tables);
        for (auto e : copy_ev) cudaEventDestroy(e);
        for (auto e : free_ev) cudaEventDestroy(e);
        for (auto s : copy_streams) cudaStreamDestroy(s);
        if (vstream) cudaStreamDestroy(vstream);
        if (done_ev) cudaEventDestroy(done_ev);
        if (entry_ev) cudaEventDestroy(entry_ev);
    }
};

static std::mutex g_ing_mu;
static std::map<FsContext*, GpuIngest*> g_ingests;

GpuIngest* gpu_ingest_get(FsContext* ctx, Err* err) {
    std::lock_guard<std::mutex> lk(g_ing_mu);
    auto it = g_ingests.find(ctx);
    if (it != g_ingests.end()) return it->second;
    GpuIngest* g = new GpuIngest();
    *err = g->init(ctx->conf.b200);
    if (*err) {
        delete g;
        return nullptr;
    }
    g_ingests[ctx] = g;
    // the arenas named in the configuration are mapped + pinned from now on, in the background, off any read path
    if (ctx->conf.b200.zero_copy && ctx->conf.b200.arena)
        for (const std::string& spec : ctx->conf.b200.arena_dirs) {
            StorageDir d;
            if (parse_data_dir(spec, &d)) continue;
            g->arena.preregister_dir((ctx->conf.cluster_id.empty() ? d.path : d.path + "/" + ctx->conf.cluster_id) + "/arena");
        }
    return g;
}

Err gpu_ingest_preregister(FsContext* ctx) {
    Err e;
    gpu_ingest_get(ctx, &e);
    return e;
}

void gpu_ingest_arena_stats(FsContext* ctx, uint64_t out[5]) {
    memset(out, 0, 5 * sizeof(uint64_t));
    std::lock_guard<std::mutex> lk(g_ing_mu);
    auto it = g_ingests.find(ctx);
    if (it == g_ingests.end()) return;
    double sec = 0;
    it->second->arena.stats(&out[0], &out[1], &sec);
    out[2] = static_cast<uint64_t>(sec * 1e6), out[3] = it->second->arena.dma_jobs.load(), out[4] = it->second->arena.dma_bytes.load();
}

void gpu_ingest_wait_registered(FsContext* ctx) {
    GpuIngest* g = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_ing_mu);
        auto it = g_ingests.find(ctx);
        if (it != g_ingests.end()) g = it->second;
    }
    if (g) g->registrar.drain(), g->arena.drain();
}

void gpu_ingest_release(FsContext* ctx) {
    std::lock_guard<std::mutex> lk(g_ing_mu);
    auto it = g_ingests.find(ctx);
    if (it == g_ingests.end()) return;
    delete it->second;
    g_ingests.erase(it);
}

// ------------------------------------------------------------------ GpuFsReader

Err GpuFsReader::open(FsContext* ctx, const std::string& path, std::unique_ptr<GpuFsReader>* out) {
    std::unique_ptr<GpuFsReader> r(new GpuFsReader());
    r->ctx_ = ctx;
    CV_RETURN_IF_ERR(ctx->ns.get_block_locations(path, &r->fbp_));
    Err e;
    r->ing_ = gpu_ingest_get(ctx, &e);
    if (e) return e;
    *out = std::move(r);
    return Err::ok();
}

GpuFsReader::~GpuFsReader() {
    if (ing_) {
        std::lock_guard<std::mutex> lk(ing_->mu);
        harvest();
        if (ing_->pending_owner == this) ing_->pending_owner = nullptr;
    }
}

Err GpuFsReader::seek(int64_t pos) {
    if (pos < 0) return Err::common("Cannot seek to negative offset");
    // past-EOF positions are legal through FsReader (FsReaderParallel::seek clamps, fs_reader_parallel.rs:175-181): reads return 0
    pos_ = pos;
    return Err::ok();
}

Err GpuFsReader::complete() {
    uint64_t s, v;
    uint32_t b;
    return verify(&s, &b, &v);
}

// every table of the per-call table image starts 256-byte aligned
static size_t table_up(size_t x) { return (x + 255) & ~size_t(255); }

// Delivery riding on a read: after the bytes landed in d_dst and were CRC'd, spans of them are copied or converted to d_out + dst_off,
// in the same launch train on the verify stream, no extra sync.  Page buffers of a FUSE reply (Reader::fuse_read +
// ResponseData::as_iovec on the device), or the spans of the boundary blocks of a vectored read: one-row spans as segs (K3), spans of
// several rows as strided (K3 over 2D descriptors), spans of converting ranges as casts (K5).  When a cast span has an FP8 source or a
// scale, `scales` (one CvScaleSeg per cast, a null scale for the others) is uploaded too and K5's scaled instance runs instead of K5.
struct GpuFsReader::Scatter {
    uint8_t* d_out;
    std::vector<CvSeg> segs;
    uint64_t total = 0;  // sum of segs[i].len
    std::vector<CvStridedSeg> strided;
    uint64_t strided_total = 0;  // sum of strided[i].len * strided[i].rows
    std::vector<CvCastSeg> casts;
    uint64_t cast_elems = 0, cast_chunks = 0;  // sum of casts[i].elems * rows, and the next segment's `first`
    std::vector<CvScaleSeg> scales;
    bool scaled = false;  // a cast span has an FP8 source or a scale

    explicit Scatter(uint8_t* out) : d_out(out) {}

    // A span of range `r`: row k < rows is `len` source bytes at d_dst + src + k * file_pitch, delivered to d_out + dst + k * dst_pitch
    // (converted when the range converts).  `file_pos` is the file offset of the span's first byte.
    void add(uint64_t src, uint64_t dst, uint64_t len, uint64_t rows, const ReadvRange& r, int64_t file_pos) {
        if (r.cast()) {
            const int64_t ss = dtype_size(r.src_dtype);
            const uint64_t elems = len / static_cast<uint64_t>(ss);
            casts.push_back(CvCastSeg{src, dst, elems, rows, static_cast<uint64_t>(r.file_pitch), static_cast<uint64_t>(r.dst_pitch), cast_chunks,
                                      r.src_dtype, r.dst_dtype});
            cast_elems += elems * rows;
            cast_chunks += rows * CV_CAST_ROW_CHUNKS(elems);
            // the view position of the span's first element: first_elem + (its file offset - file_off) / src size
            const ReadvScale& g = r.scale;
            scales.push_back(r.scaled() ? CvScaleSeg{g.ptr, uint64_t(g.block_rows), uint64_t(g.block_cols), uint64_t(g.cols), uint64_t(g.view_cols),
                                                     uint64_t(g.first_elem + (file_pos - r.file_off) / ss), uint64_t(r.file_pitch / ss), g.dtype, 0}
                                        : CvScaleSeg{});
            scaled |= r.scaled() || is_f8(r.src_dtype);
        } else if (rows == 1) {
            segs.push_back(CvSeg{src, dst, len});
            total += len;
        } else {
            strided.push_back(CvStridedSeg{src, dst, len, rows, static_cast<uint64_t>(r.file_pitch), static_cast<uint64_t>(r.dst_pitch)});
            strided_total += len * rows;
        }
    }

    // The scatter's section of the per-call tables: segs | strided | casts | scales (when scaled).  [k] = where table k starts, [4] = bytes.
    std::array<size_t, 5> offsets() const {
        std::array<size_t, 5> o{};
        o[1] = table_up(sizeof(CvSeg) * segs.size());
        o[2] = o[1] + table_up(sizeof(CvStridedSeg) * strided.size());
        o[3] = o[2] + table_up(sizeof(CvCastSeg) * casts.size());
        o[4] = o[3] + (scaled ? table_up(sizeof(CvScaleSeg) * scales.size()) : 0);
        return o;
    }
    size_t bytes() const { return offsets()[4]; }
    template <typename T>
    T* table(uint8_t* section, int k) const { return reinterpret_cast<T*>(section + offsets()[k]); }

    // the tables into the section's pinned image
    void write(uint8_t* h) const {
        std::copy(segs.begin(), segs.end(), table<CvSeg>(h, 0));
        std::copy(strided.begin(), strided.end(), table<CvStridedSeg>(h, 1));
        std::copy(casts.begin(), casts.end(), table<CvCastSeg>(h, 2));
        if (scaled) std::copy(scales.begin(), scales.end(), table<CvScaleSeg>(h, 3));
    }

    // K3, K3 over 2D descriptors, then K5 or its scaled instance, out of d_src with the tables uploaded at d; a kind without spans
    // launches nothing
    Err launch(const uint8_t* d_src, uint8_t* d, cudaStream_t s) const {
        if (!segs.empty()) CVK_TRY(cvk_gather_pages(d_src, table<CvSeg>(d, 0), static_cast<uint32_t>(segs.size()), total, d_out, s));
        if (!strided.empty()) CVK_TRY(cvk_gather_strided(d_src, table<CvStridedSeg>(d, 1), static_cast<uint32_t>(strided.size()), strided_total, d_out, s));
        const uint32_t n_casts = static_cast<uint32_t>(casts.size());
        if (n_casts && scaled) CVK_TRY(cvk_gather_cast_scaled(d_src, table<CvCastSeg>(d, 2), table<CvScaleSeg>(d, 3), n_casts, cast_elems, d_out, s));
        else if (n_casts) CVK_TRY(cvk_gather_cast(d_src, table<CvCastSeg>(d, 2), n_casts, cast_elems, d_out, s));
        return Err::ok();
    }
};

Err GpuFsReader::fuse_read_device(int64_t want, void* d_scratch, void* d_page_base, const uint64_t* page_offsets, int64_t n_pages, int64_t page_size,
                                   void* stream, int64_t* n) {
    *n = 0;
    if (page_size <= 0) return Err::common("page_size must be positive");
    const int64_t take = std::max<int64_t>(0, std::min(want, len() - pos_));
    const int64_t need_pages = (take + page_size - 1) / page_size;
    if (need_pages > n_pages) return Err::common("not enough page buffers for the reply");
    Scatter ps(static_cast<uint8_t*>(d_page_base));
    const ReadvRange bytes{};  // a page is one row of a plain byte range
    for (int64_t i = 0; i < need_pages; i++)
        ps.add(static_cast<uint64_t>(i * page_size), page_offsets[i], static_cast<uint64_t>(std::min(page_size, take - i * page_size)), 1, bytes, 0);
    return read_device_impl(d_scratch, take, stream, n, &ps);
}

Err GpuFsReader::read_device(void* d_dst, int64_t cap, void* stream, int64_t* n) { return read_device_impl(d_dst, cap, stream, n, nullptr); }

Err GpuFsReader::read_device_impl(void* d_dst, int64_t cap, void* stream, int64_t* n, const Scatter* scatter) {
    *n = 0;
    const int64_t end = std::min(len(), pos_ + std::max<int64_t>(cap, 0));
    if (end <= pos_) return Err::ok();
    std::vector<Job> jobs;
    int64_t p = pos_;
    while (p < end) {
        int64_t boff;
        size_t idx;
        CV_RETURN_IF_ERR((*fbp_).get_read_block(p, &boff, &idx));
        const int64_t blen = (*fbp_).block_locs[idx].block.len;
        const int64_t take = std::min(end - p, blen - boff);
        jobs.push_back(Job{&(*fbp_).block_locs[idx], boff, take, p - pos_, boff == 0 && take == blen});
        p += take;
    }
    CV_RETURN_IF_ERR(run_jobs(jobs, static_cast<uint8_t*>(d_dst), stream, scatter));
    *n = end - pos_;
    pos_ = end;
    return Err::ok();
}

Err GpuFsReader::read_device_sharded(int rank, int world, void* d_dst, int64_t cap, void* stream, int64_t* n) {
    *n = 0;
    std::vector<ShardJob> plan;
    int64_t total = 0;
    CV_RETURN_IF_ERR(plan_shard(*fbp_, rank, world, cap, &plan, &total));
    std::vector<Job> jobs;
    for (const auto& p : plan) jobs.push_back(Job{&(*fbp_).block_locs[p.block], 0, p.len, p.dst_off, true});
    CV_RETURN_IF_ERR(run_jobs(jobs, static_cast<uint8_t*>(d_dst), stream));
    *n = total;
    return Err::ok();
}

namespace {

// Wait for `cond()`: a short spin, then sleep in growing steps so waiting threads do not starve the worker threads.
template <typename F>
static inline void backoff_wait(F cond) {
    for (int i = 0; i < 64; i++) {
        if (cond()) return;
        std::this_thread::yield();
    }
    unsigned us = 10;
    while (!cond()) {
        usleep(us);
        if (us < 200) us *= 2;
    }
}

}  // namespace

enum JobMode : uint8_t { kPlain = 0, kFramed = 1, kHole = 3 };

// n bytes of the file at `path` from file_off -> buf
static Err pread_full(const std::string& path, int64_t file_off, uint8_t* buf, int64_t n) {
    const int fd = ::open(path.c_str(), O_RDONLY | O_CLOEXEC);
    if (fd < 0) return Err::io(str_printf("open %s: %s", path.c_str(), strerror(errno)));
    Err e;
    for (int64_t got = 0; got < n && !e;) {
        const ssize_t r = pread(fd, buf + got, static_cast<size_t>(n - got), file_off + got);
        if (r < 0 && errno == EINTR) continue;
        if (r <= 0) e = Err::io(str_printf("read block file: %s", r == 0 ? "unexpected eof" : strerror(errno)));
        else got += r;
    }
    ::close(fd);
    return e;
}

// fn(connection) on each replica of `lb` in turn until one succeeds (a pooled `conn` to the replica is reused while it is healthy);
// -> the last error when none did.
template <typename F>
static Err for_each_replica(FsContext* ctx, const LocatedBlock& lb, std::unique_ptr<BlockClient>* conn, F fn) {
    Err last = ctx->no_available_worker(lb.locs);
    for (const WorkerAddress& loc : lb.locs) {
        last = ctx->connection_to(loc, conn);
        if (!last) last = fn(conn->get());
        if (!last) return Err::ok();
    }
    return last;
}

// Open(short_circuit=true) on connection `c`: the worker names the block file (and, for an arena block, the extent inside it)
static Err open_on(FsContext* ctx, BlockClient* c, const LocatedBlock& lb, int64_t block_off, int64_t req_id, BlockReadResponse* resp) {
    CV_RETURN_IF_ERR(c->open_block(ctx->conf.client, lb.block, block_off, lb.block.len, req_id, 0, true, ctx->read_chunk_size(), resp, ctx->conf.b200.arena));
    return resp->has_path ? Err::ok() : Err::common("read_context.path is none");
}

// Fetch one job's bytes into `slot`.
//   kPlain   short-circuit: payload only (pread of the block file the worker named)
//   kFramed  verbatim: the response stream exactly as received: 22-byte prefixes + payloads (unpacked on the GPU by K2, which
//            also clips the last chunk of a range that stops short of the block end)
// A replica whose block file cannot be read is given up for the next one.
static Err fetch_job(FsContext* ctx, const LocatedBlock& lb, int64_t block_off, int64_t n, JobMode mode, int64_t chunk, uint8_t* slot,
                     std::unique_ptr<BlockClient>* conn, int64_t* req_id_out, size_t* wire_bytes) {
    return for_each_replica(ctx, lb, conn, [&](BlockClient* c) -> Err {
        const int64_t req_id = new_req_id();
        *req_id_out = req_id;
        BlockReadResponse resp;
        if (mode == kPlain) {
            CV_RETURN_IF_ERR(open_on(ctx, c, lb, block_off, req_id, &resp));
            CV_RETURN_IF_ERR(pread_full(resp.path, (resp.has_arena ? resp.arena_off : 0) + block_off, slot, n));  // arena block: an extent of the segment file
            *wire_bytes = static_cast<size_t>(n);
            return c->read_commit_deferred(lb.block, req_id, 1);  // its answer is consumed in front of this connection's next request
        }
        // Open + every Running request + Complete in one write (the worker serves them in order, read_handler.rs:60-207).  The
        // worker answers each Running with min(chunk, block_len - pos) bytes, so the last frame of a range that stops short of
        // the block end carries bytes past it: they are received like the rest and clipped by K2 (CvStreamDesc.tail_clip).
        const int64_t nfr = (n + chunk - 1) / chunk;
        int64_t left = std::min<int64_t>(nfr * chunk, lb.block.len - block_off);  // payload bytes on the wire
        CV_RETURN_IF_ERR(c->send_block_read_pipeline(ctx->conf.client, lb.block, block_off, req_id, chunk, nfr, &resp));
        uint8_t* w = slot;
        Err e;
        for (int64_t f = 0; f < nfr && !e; f++) {
            e = recv_exact(c->fd(), w, kProtocolSize);
            Protocol p;
            if (!e) e = decode_protocol(w, &p);
            if (e) break;
            const int64_t want = std::min(chunk, left);
            if (!p.is_success() || p.header_len != 0 || p.data_len != want) {
                // error response (or an unexpected chunk): drain this frame, report it, drop the connection
                std::string body(static_cast<size_t>(p.header_len + p.data_len), '\0');
                if (!body.empty() && recv_exact(c->fd(), &body[0], body.size())) c->broken = true;
                e = p.is_success() ? Err::common(str_printf("unexpected chunk length %d, expected %lld", p.data_len, (long long)want))
                                   : decode_error_body(reinterpret_cast<const uint8_t*>(body.data()) + p.header_len, static_cast<size_t>(p.data_len));
                break;
            }
            e = recv_exact(c->fd(), w + kProtocolSize, static_cast<size_t>(want));
            w += kProtocolSize + want, left -= want;
        }
        if (e) {
            c->broken = true;  // responses of the remaining pipelined requests may still be in flight
            return e;
        }
        *wire_bytes = static_cast<size_t>(w - slot);
        return Err::ok();  // the Complete went out with the rest; its answer is consumed in front of this connection's next request
    });
}

// Open(short_circuit=true) on the first replica that answers; returns the block file path.
static Err open_short_circuit(FsContext* ctx, const LocatedBlock& lb, int64_t block_off, std::unique_ptr<BlockClient>* conn, int64_t* req_id,
                              BlockReadResponse* out) {
    return for_each_replica(ctx, lb, conn, [&](BlockClient* c) {
        *req_id = new_req_id();
        return open_on(ctx, c, lb, block_off, *req_id, out);
    });
}

// Pull the last call's per-block CRCs / mismatch count / frame flags (already copied to the pinned mirror on vstream).
Err GpuFsReader::harvest() {
    if (!pending_.active) return Err::ok();
    GpuIngest& G = *ing_;
    cudaSetDevice(G.device);
    CU_TRY(cudaStreamSynchronize(G.vstream));
    const TableLayout& tl = pending_.tl;
    uint32_t* crc = reinterpret_cast<uint32_t*>(G.h_result);
    for (size_t j = pending_.f0; j < pending_.f1; j++) sum_crc_ += crc[j];
    n_verified_ += pending_.n_compared;
    stats_.verified += pending_.n_compared;
    n_bad_ += *tl.nbad(crc);
    const uint32_t* ferr = tl.ferr(crc);
    for (size_t f = 0; f < tl.F; f++)
        if (ferr[f]) {
            n_bad_frames_++;
            if (!first_frame_err_) first_frame_err_ = ferr[f];
        }
    pending_.active = false;
    held_maps_.clear();  // every copy that read from these mappings has completed (vstream waited on them)
    if (G.pending_owner == this) G.pending_owner = nullptr;
    if (n_bad_frames_) return Err(kAbnormalData, str_printf("%llu frame prefixes failed validation (first flags 0x%x)", (unsigned long long)n_bad_frames_, first_frame_err_));
    return Err::ok();
}

Err GpuFsReader::verify(uint64_t* sum_crc, uint32_t* n_bad, uint64_t* n_verified) {
    Err e;
    if (ing_) {
        std::lock_guard<std::mutex> lk(ing_->mu);
        e = harvest();
    }
    *sum_crc = sum_crc_, *n_bad = n_bad_, *n_verified = n_verified_;
    return e;
}

// `p` must be device memory on `device`
static Err check_device_dst(const void* p, int device) {
    cudaPointerAttributes pa;
    if (cudaPointerGetAttributes(&pa, p) != cudaSuccess || pa.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        return Err::common("cv_read_device: destination is not device memory");
    }
    if (pa.device != device) return Err::common(str_printf("cv_read_device: destination lives on device %d but [b200] device = %d", pa.device, device));
    return Err::ok();
}

GpuFsReader::TableLayout::TableLayout(size_t j, size_t f, size_t scatter_bytes) : J(j), F(f) {
    const auto up = table_up;
    o_len = up(8 * J), o_exp = up(o_len + 8 * J), o_skip = up(o_exp + 4 * J), o_scatter = up(o_skip + J), o_crc = up(o_scatter + scatter_bytes);
    o_streams = up(o_crc + 4 * res_words()), o_fdesc = up(o_streams + sizeof(CvStreamDesc) * J);
    bytes = up(o_fdesc + sizeof(CvFrameDesc) * F);
}

// What one run_jobs call does, decided before any CUDA call.
struct GpuFsReader::CallPlan {
    std::vector<JobMode> mode;             // per job
    bool call_framed = false;              // a block without a local replica (or short_circuit off): every job runs framed
    bool any_verbatim = false;             // some job is received verbatim (framed) and unpacked by K2
    std::vector<int64_t> wire_payload;     // framed jobs: payload bytes the worker sends (>= n when the range stops short of the block end)
    std::vector<uint32_t> first_frame;     // [J + 1]: first frame of each job
    size_t F = 0;                          // frames in the call
    size_t need_slot = 0;                  // pinned-slot bytes the largest job needs
    int64_t chunk = 0;                     // framed chunk size
    size_t k = 1, NG = 0, NS = 0;          // jobs per copy group, copy groups in the call, super-slots in the ring
    size_t vgroups = 1, B = 1;             // copy groups per verify launch, and the jobs they hold
    std::vector<uint8_t> group_verbatim;   // per copy group: holds a framed job
    int T_threads = 1;                     // fetch workers
    TableLayout tl;
};

Err GpuFsReader::plan_call(const std::vector<Job>& jobs, size_t scatter_bytes, CallPlan* out) const {
    CallPlan& P = *out;
    const B200Conf& bc = ctx_->conf.b200;
    const size_t J = jobs.size();
    P.chunk = std::min<int64_t>(std::max<int64_t>(bc.gpu_chunk_size, 4096), kMaxDataSize);
    // Short-circuit (the reference default for a same-host worker, client_conf.rs:339) only when every block of this call has a local
    // replica; otherwise the whole call runs framed (any worker serves those).
    P.mode.assign(J, kPlain);
    for (size_t j = 0; j < J; j++) {
        const LocatedBlock& lb = *jobs[j].lb;
        if (lb.locs.empty()) {
            if (!lb.block.has_alloc_opts) return ctx_->no_available_worker(lb.locs);
            P.mode[j] = kHole;
            continue;
        }
        bool local = false;
        for (const auto& a : lb.locs) local |= ctx_->is_local_worker(a);
        if (!(ctx_->conf.client.short_circuit && local)) P.call_framed = true;
    }
    P.first_frame.assign(J + 1, 0);
    P.wire_payload.assign(J, 0);
    for (size_t j = 0; j < J; j++) {
        P.first_frame[j] = static_cast<uint32_t>(P.F);
        size_t bytes = static_cast<size_t>(jobs[j].n);
        if (P.mode[j] != kHole && P.call_framed) {
            // every framed job is received verbatim and unpacked by K2; a range that stops short of its block's end gets the
            // worker's whole last chunk and K2 clips it (CvStreamDesc.tail_clip) -- no host-side unpacking anywhere
            P.mode[j] = kFramed;
            const int64_t nfr = (jobs[j].n + P.chunk - 1) / P.chunk;
            P.wire_payload[j] = std::min<int64_t>(nfr * P.chunk, jobs[j].lb->block.len - jobs[j].block_off);
            bytes = static_cast<size_t>(P.wire_payload[j] + nfr * kProtocolSize);
            P.F += static_cast<size_t>(nfr);
            P.any_verbatim = true;
        }
        P.need_slot = std::max(P.need_slot, bytes);
    }
    P.first_frame[J] = static_cast<uint32_t>(P.F);
    // copy groups: k consecutive jobs share one super-slot and, when they are contiguous, one cudaMemcpyAsync
    P.k = static_cast<size_t>(std::max(1, std::min(bc.copy_group, ing_->nslots / 4)));
    P.NG = (J + P.k - 1) / P.k;
    P.NS = static_cast<size_t>(ing_->nslots) / P.k;
    P.vgroups = std::max<size_t>(1, (static_cast<size_t>(std::max(1, bc.verify_batch)) + P.k - 1) / P.k);
    P.B = P.vgroups * P.k;
    P.group_verbatim.assign(P.NG, 0);
    for (size_t j = 0; j < J; j++) P.group_verbatim[j / P.k] |= P.mode[j] == kFramed;
    P.T_threads = static_cast<int>(std::min<size_t>(static_cast<size_t>(std::max(1, bc.fetch_threads)), P.NG));
    P.tl = TableLayout(J, P.F, scatter_bytes);
    return Err::ok();
}

namespace {

// Host-to-device copies of (dst, src, len) pieces on one stream.  A piece that continues the previous one in the source AND in the
// destination extends it, so one cudaMemcpyAsync moves both -- except across a register slice of an arena segment: a copy never spans
// two separately registered slices.
struct H2D {
    cudaStream_t cs;
    uint64_t* counted;  // bytes enqueued (the reader's h2d_bytes)
    uint8_t* dst = nullptr;
    const uint8_t* src = nullptr;
    size_t len = 0;
    bool pending = false;
    const ArenaSeg* seg = nullptr;  // the pending piece's source lies in this segment
    cudaError_t ce = cudaSuccess;

    H2D(cudaStream_t s, uint64_t* c) : cs(s), counted(c) {}
    bool ok() const { return ce == cudaSuccess; }
    void add(uint8_t* d, const uint8_t* s, size_t n, const ArenaSeg* sg = nullptr) {
        if (pending && sg == seg && d == dst + len && s == src + len) {
            len += n;
            return;
        }
        flush();
        dst = d, src = s, len = n, seg = sg, pending = true;
    }
    void flush() {
        if (!pending || !ok()) return;
        for (size_t done = 0; done < len && ok();) {
            size_t piece = len - done;
            if (seg) {
                const size_t in_seg = static_cast<size_t>(src - seg->base) + done;
                piece = std::min(piece, (in_seg / seg->slice + 1) * seg->slice - in_seg);
            }
            ce = cudaMemcpyAsync(dst + done, src + done, piece, cudaMemcpyHostToDevice, cs);
            done += piece;
        }
        *counted += len;
        pending = false;
    }
    Err finish() {
        flush();
        return ok() ? Err::ok() : Err::io(str_printf("H2D enqueue: %s", cudaGetErrorString(ce)));
    }
};

}  // namespace

// One run_jobs call in flight: its tables, the fetch workers, the super-slot handoff between them and the verifier, the ingest paths a
// copy group can take, the verifier and the finish.  Each ingest path returns Err::ok() when the group's copies are enqueued,
// kUnsupported when the group must go to the next path (GDS -> registered mappings / arena -> pinned ring), or the error that fails the
// call.
struct GpuFsReader::Call {
    struct Group {
        size_t g, j0, j1;  // copy group, its jobs [j0, j1)
        int t;             // fetch worker
        cudaStream_t cs;
    };
    GpuFsReader& r;
    GpuIngest& G;
    const std::vector<Job>& jobs;
    const CallPlan& P;
    uint8_t* d_dst;
    const Scatter* scatter;
    size_t f0 = 0, f1 = 0, n_compared = 0;  // write_tables: CRCs of jobs [f0, f1) are summed, n_compared of them compared
    bool compare = false;                   // with the manifest, by cvk_verify_crcs_masked
    std::atomic<size_t> next_group{0};
    std::atomic<bool> abort{false};
    std::mutex err_mu, held_mu;
    Err err;
    std::vector<std::atomic<int>> copied;        // per copy group: published
    std::vector<std::atomic<int64_t>> released;  // per super-slot: last copy group whose release event is recorded
    std::vector<int64_t> req_ids;
    std::atomic<bool> use_mapped, use_gds;
    std::atomic<uint64_t> gds_bytes{0};
    std::vector<double> fetch_sec;
    std::vector<uint64_t> h2d;
    std::once_flag ring_once;
    Err ring_err;

    Call(GpuFsReader& reader, const std::vector<Job>& js, const CallPlan& plan, uint8_t* dst, const Scatter* sc)
        : r(reader), G(*reader.ing_), jobs(js), P(plan), d_dst(dst), scatter(sc), copied(plan.NG), released(plan.NS), req_ids(js.size(), 0),
          fetch_sec(static_cast<size_t>(plan.T_threads), 0.0), h2d(static_cast<size_t>(plan.T_threads), 0) {
        const B200Conf& bc = r.ctx_->conf.b200;
        for (auto& c : copied) c.store(0);
        for (auto& x : released) x.store(-1);
        use_mapped.store(bc.zero_copy);
        bool any_disk = false;  // cuFile is probed only by a read that has disk-tier blocks
        for (size_t j = 0; j < jobs.size() && !any_disk; j++) any_disk = jobs[j].lb->block.storage_type != kStorageMem;
        use_gds.store(!P.call_framed && bc.gds != 0 && any_disk && gds_info().available);
    }
    void fail(const Err& e) {
        std::lock_guard<std::mutex> lk(err_mu);
        if (!err) err = e;
        abort.store(true);
    }
    // the pinned ring (and the device staging ring for verbatim frames) is only materialised when a group needs it: the zero-copy
    // path never touches it
    Err ensure_ring() {
        std::call_once(ring_once, [&] { ring_err = G.ensure(P.need_slot, P.any_verbatim); });
        return ring_err;
    }

    void worker(int t, bool own_thread) {
        if (own_thread) bind_cpus(G.cpus);  // an inline call (single copy group: small reads) must not re-pin the caller
        cudaSetDevice(G.device);
        cudaStream_t cs = G.copy_streams[static_cast<size_t>(t) % G.copy_streams.size()];
        std::unique_ptr<BlockClient> conn;
        for (;;) {
            const size_t g = next_group.fetch_add(1);
            if (g >= P.NG || abort.load()) break;
            const Group gr{g, g * P.k, std::min(jobs.size(), g * P.k + P.k), t, cs};
            if (!acquire_slot(gr)) break;
            bool all_plain = true, all_disk = true;
            for (size_t j = gr.j0; j < gr.j1; j++) {
                all_plain = all_plain && P.mode[j] == kPlain;
                all_disk = all_disk && jobs[j].lb->block.storage_type != kStorageMem;
            }
            Err e(kUnsupported, "");  // kUnsupported: the group goes to the next path
            if (all_plain && all_disk && use_gds.load(std::memory_order_relaxed)) {
                e = fetch_group_gds(gr, &conn);
                if (e.kind == kUnsupported) use_gds.store(false);  // this file system / this box cannot do it: the next path redoes the group
            }
            if (e.kind == kUnsupported && all_plain && use_mapped.load(std::memory_order_relaxed)) {
                e = fetch_group_mapped(gr, &conn);
                if (e.kind == kUnsupported) use_mapped.store(false);  // cannot register file mappings here: the pinned ring takes over
            }
            if (e.kind == kUnsupported) e = fetch_group_ring(gr, &conn);
            if (!publish(gr, e)) break;
        }
        if (conn) {
            // multi-group reads: settle the deferred Completes here (their answers are long in); a single-group read (the
            // latency path, C5) parks the connection with its last answer outstanding and the next request consumes it
            if (P.NG > 1) conn->drain_pending();
            r.ctx_->release(std::move(conn));
        }
    }

    // ---- The super-slot handoff.  Copy group g owns super-slot super_slot(g) of the pinned ring and of its device mirror d_stage: k
    // slots of slot_bytes, job j's own slot at slot_off(j) in both.  A super-slot serves every NS-th group.  Every group takes part
    // whichever path moved it (arena, mapped and GDS groups too): copy_ev belongs to the super-slot, not to a path.  Nothing but these
    // four operations touches copy_ev, free_ev, released or copied.
    size_t super_slot(size_t g) const { return g % P.NS; }
    size_t slot_off(size_t j) const { return (super_slot(j / P.k) * P.k + j % P.k) * G.slot_bytes; }

    // Fetch worker, before the group: wait until the super-slot's previous tenant has been released, then for that tenant's copies (or,
    // for a verbatim group, its K2) to finish with the slot.
    bool acquire_slot(const Group& gr) {
        if (gr.g < P.NS) return true;
        const size_t ss = super_slot(gr.g);
        const int64_t want = static_cast<int64_t>(gr.g - P.NS);
        backoff_wait([&] { return released[ss].load(std::memory_order_acquire) >= want || abort.load(); });
        if (abort.load()) return false;
        cudaEventSynchronize(P.group_verbatim[gr.g - P.NS] ? G.free_ev[ss] : G.copy_ev[ss]);
        return true;
    }

    // Fetch worker, after the group: hand it to the verifier once its copies are enqueued.  A verbatim group's super-slot is released
    // by the verifier after K2 has unpacked it (release_verbatim); every other group's as soon as its copy event is recorded.
    bool publish(const Group& gr, const Err& e) {
        const size_t ss = super_slot(gr.g);
        const cudaError_t ce = e ? cudaSuccess : cudaEventRecord(G.copy_ev[ss], gr.cs);
        if (e || ce != cudaSuccess) {
            fail(e ? e : Err::io(str_printf("event record: %s", cudaGetErrorString(ce))));
            return false;
        }
        if (!P.group_verbatim[gr.g]) released[ss].store(static_cast<int64_t>(gr.g), std::memory_order_release);
        copied[gr.g].store(1, std::memory_order_release);
        return true;
    }

    // Verifier, before a batch: wait until groups [v0, v1) are published, then order vstream after their copies.  false: the call failed.
    bool await_copies(size_t v0, size_t v1) {
        for (size_t g = v0; g < v1; g++)
            backoff_wait([&] { return copied[g].load(std::memory_order_acquire) != 0 || abort.load(); });
        if (abort.load()) return false;
        for (size_t g = v0; g < v1; g++) cudaStreamWaitEvent(G.vstream, G.copy_ev[super_slot(g)], 0);
        return true;
    }

    // Verifier, after a batch's K2: release the super-slots of its verbatim groups.
    void release_verbatim(size_t v0, size_t v1) {
        for (size_t g = v0; g < v1; g++)
            if (P.group_verbatim[g]) {
                cudaEventRecord(G.free_ev[super_slot(g)], G.vstream);
                released[super_slot(g)].store(static_cast<int64_t>(g), std::memory_order_release);
            }
    }

    // GPUDirect Storage: blocks of a disk tier go file -> HBM by cuFileRead, no host ring
    Err fetch_group_gds(const Group& gr, std::unique_ptr<BlockClient>* conn) {
        const double t0 = now_sec();
        backoff_wait([&] { return cudaEventQuery(G.entry_ev) != cudaErrorNotReady; });  // cuFile knows nothing of the caller's stream
        Err e;
        for (size_t j = gr.j0; j < gr.j1 && !e; j++) {
            const Job& job = jobs[j];
            BlockReadResponse resp;
            int64_t rid = 0;
            e = open_short_circuit(r.ctx_, *job.lb, job.block_off, conn, &rid, &resp);
            if (!e) e = gds_read(resp.path, d_dst + job.dst_off, job.n, (resp.has_arena ? resp.arena_off : 0) + job.block_off);
            if (!e) e = (*conn)->read_commit_deferred(job.lb->block, rid, 1);
            if (!e) gds_bytes += static_cast<uint64_t>(job.n);
        }
        fetch_sec[static_cast<size_t>(gr.t)] += now_sec() - t0;
        return e;
    }

    // Zero-copy: DMA out of the mem arena's pinned segments, or out of registered mmaps of the block files.  Groups whose mappings
    // are not ready (or cannot be pinned) are pread out of the block files into the ring.
    Err fetch_group_mapped(const Group& gr, std::unique_ptr<BlockClient>* conn) {
        const double t0 = now_sec();
        const size_t n = gr.j1 - gr.j0;
        std::vector<std::string> paths(n);
        std::vector<int64_t> lens(n), rids(n), base_offs(n, 0);
        size_t n_arena = 0;
        Err e;
        std::vector<BlockReadResponse> resps;
        if (!open_group_batched(gr, conn, &rids, &resps)) {  // one Open round trip per block, with failover to the other replicas
            resps.assign(n, BlockReadResponse());
            for (size_t i = 0; i < n && !e; i++) {
                const Job& job = jobs[gr.j0 + i];
                e = open_short_circuit(r.ctx_, *job.lb, job.block_off, conn, &rids[i], &resps[i]);
            }
        }
        for (size_t i = 0; i < n; i++) {
            paths[i] = resps[i].path, lens[i] = jobs[gr.j0 + i].lb->block.len;
            if (resps[i].has_arena) base_offs[i] = resps[i].arena_off, n_arena++;
        }
        bool via_ring = n_arena > 0;  // arena extents (mixed group, or segments that cannot be pinned): pread out of the segment file
        if (!e && n_arena == n && !G.arena.unsupported.load(std::memory_order_relaxed)) {
            e = fetch_arena(gr, paths, base_offs, rids, conn);
            if (e.kind != kUnsupported) {
                fetch_sec[static_cast<size_t>(gr.t)] += now_sec() - t0;
                return e;
            }
            e = Err::ok();  // segments cannot be pinned here: the group goes through the ring
        }
        std::shared_ptr<RegMapping> m;
        if (!e && !via_ring) e = find_mapping(paths, lens, &m, &via_ring);
        H2D q(gr.cs, &h2d[static_cast<size_t>(gr.t)]);
        if (!e && via_ring) {
            e = ensure_ring();
            if (!e) e = fill_ring(gr, q, [&](size_t j, uint8_t* at, size_t* wire) {
                    *wire = static_cast<size_t>(jobs[j].n);
                    return pread_full(paths[j - gr.j0], base_offs[j - gr.j0] + jobs[j].block_off, at, jobs[j].n);
                });
        } else if (!e) {
            size_t moff = 0;  // the group's block files lie back to back in the mapping, each page-rounded
            for (size_t i = 0; i < n; i++) {
                const Job& job = jobs[gr.j0 + i];
                q.add(d_dst + job.dst_off, m->base + moff + job.block_off, static_cast<size_t>(job.n));
                moff += page_up(static_cast<size_t>(lens[i]));
            }
            std::lock_guard<std::mutex> lk(held_mu);
            r.held_maps_.push_back(m);
        }
        const Err copy_err = e ? Err::ok() : q.finish();
        for (size_t j = gr.j0; j < gr.j1 && !e; j++) e = (*conn)->read_commit(jobs[j].lb->block, rids[j - gr.j0], 1);
        fetch_sec[static_cast<size_t>(gr.t)] += now_sec() - t0;
        return e ? e : copy_err;
    }

    // The group's Opens in one write and one round trip, on a connection to the first replica of its blocks when they all share it.
    // false: not done (blocks on different first replicas, no connection, an error or a block file the worker did not name): the
    // connection is broken if anything was sent, and the per-block path redoes the Opens on a fresh one, failover included.
    bool open_group_batched(const Group& gr, std::unique_ptr<BlockClient>* conn, std::vector<int64_t>* rids, std::vector<BlockReadResponse>* resps) {
        const WorkerAddress& a = jobs[gr.j0].lb->locs[0];  // plain jobs have a replica
        std::vector<BlockClient::OpenReq> reqs;
        for (size_t j = gr.j0; j < gr.j1; j++) {
            if (!(jobs[j].lb->locs[0] == a)) return false;
            reqs.push_back(BlockClient::OpenReq{&jobs[j].lb->block, jobs[j].block_off, new_req_id()});
        }
        if (r.ctx_->connection_to(a, conn)) return false;
        if ((*conn)->open_blocks(r.ctx_->conf.client, reqs, r.ctx_->read_chunk_size(), r.ctx_->conf.b200.arena, resps)) return false;
        for (const BlockReadResponse& x : *resps)
            if (!x.has_path) {
                (*conn)->broken = true;  // the per-block path reports it ("read_context.path is none") or fails over
                return false;
            }
        for (size_t i = 0; i < reqs.size(); i++) (*rids)[i] = reqs[i].req_id;
        return true;
    }

    // Every block of the group is an extent of an arena segment this context pinned once.  kUnsupported: a segment cannot be pinned.
    Err fetch_arena(const Group& gr, const std::vector<std::string>& paths, const std::vector<int64_t>& base_offs, const std::vector<int64_t>& rids,
                    std::unique_ptr<BlockClient>* conn) {
        std::vector<std::shared_ptr<ArenaSeg>> segs(paths.size());
        for (size_t i = 0; i < paths.size(); i++) {
            const Job& job = jobs[gr.j0 + i];
            if (i > 0 && paths[i] == paths[i - 1]) segs[i] = segs[i - 1];
            else CV_RETURN_IF_ERR(G.arena.get(paths[i], &segs[i]));
            if (static_cast<size_t>(base_offs[i] + job.block_off + job.n) > segs[i]->bytes) return Err::io("arena extent lies outside its segment");
        }
        H2D q(gr.cs, &h2d[static_cast<size_t>(gr.t)]);
        for (size_t i = 0; i < paths.size(); i++) {
            const Job& job = jobs[gr.j0 + i];
            q.add(d_dst + job.dst_off, segs[i]->base + base_offs[i] + job.block_off, static_cast<size_t>(job.n), segs[i].get());
        }
        const Err copy_err = q.finish();
        std::vector<BlockClient::OpenReq> done;  // the group's Completes in one write, answered in front of the next request
        for (size_t j = gr.j0; j < gr.j1; j++) done.push_back(BlockClient::OpenReq{&jobs[j].lb->block, jobs[j].block_off, rids[j - gr.j0]});
        const Err e = (*conn)->read_commit_deferred(done);
        if (e || copy_err) return e ? e : copy_err;
        G.arena.dma_jobs += gr.j1 - gr.j0;
        for (size_t j = gr.j0; j < gr.j1; j++) G.arena.dma_bytes += static_cast<uint64_t>(jobs[j].n);
        return Err::ok();
    }

    // The registered mapping of the group's block files: a cache hit, or registered now when the cache does the registration inline.
    // *via_ring when the group goes through the ring this time (cache full of young mappings, or registration left to the background).
    Err find_mapping(const std::vector<std::string>& paths, const std::vector<int64_t>& lens, std::shared_ptr<RegMapping>* m, bool* via_ring) {
        std::string key;
        for (const auto& p : paths) key += p, key += '|';
        std::vector<uint64_t> stamps;
        if (stat_stamps(paths, &stamps)) *m = G.reg.find(key, stamps);
        if (*m) return Err::ok();
        G.reg.misses++;
        if (G.registrar.unsupported.load()) return Err(kUnsupported, "cudaHostRegister of file mappings is not supported here");
        size_t group_bytes = 0;
        for (int64_t l : lens) group_bytes += page_up(static_cast<size_t>(l));
        if (G.reg.capacity > 0 && !G.reg.can_admit(group_bytes)) {
            // the cache is full of mappings in use or used moments ago (a scan larger than the cache): registering this group would be
            // paid for and thrown away -- it goes through the ring, now and next time
            G.reg.rejected++;
            *via_ring = true;
        } else if (G.register_inline) {
            CV_RETURN_IF_ERR(map_and_register(paths, lens, m, &stamps));
            (*m)->key = key;
            G.reg.insert(*m);
        } else {  // cold group: register it in the background for the next pass, move it through the ring now
            G.registrar.submit(Registrar::Job{key, paths, lens});
            *via_ring = true;
        }
        return Err::ok();
    }

    // The pinned ring: each job is fetched into the group's super-slot and copied from there (holes are zero-filled on the device).
    Err fetch_group_ring(const Group& gr, std::unique_ptr<BlockClient>* conn) {
        CV_RETURN_IF_ERR(ensure_ring());
        H2D q(gr.cs, &h2d[static_cast<size_t>(gr.t)]);
        CV_RETURN_IF_ERR(fill_ring(gr, q, [&](size_t j, uint8_t* at, size_t* wire) {
            const Job& job = jobs[j];
            const double t0 = now_sec();
            Err e = fetch_job(r.ctx_, *job.lb, job.block_off, job.n, P.mode[j], P.chunk, at, conn, &req_ids[j], wire);
            fetch_sec[static_cast<size_t>(gr.t)] += now_sec() - t0;
            return e ? e.ctx(str_printf("block %lld", (long long)job.lb->block.id)) : e;
        }));
        return q.finish();
    }

    // Slot layout of a ring group: when its jobs are all plain, back to back in the destination and fit into the super-slot, they
    // mirror the destination layout there and one copy moves the group; otherwise each job has a slot (and a copy) of its own.
    // fetch(j, at, &wire) puts job j's bytes at `at`; a verbatim group's frames go to the same offsets of the device staging in one copy
    // after the last.
    template <typename Fetch>
    Err fill_ring(const Group& gr, H2D& q, Fetch fetch) {
        const Job& first = jobs[gr.j0];
        const Job& last = jobs[gr.j1 - 1];
        bool mirror = static_cast<size_t>(last.dst_off + last.n - first.dst_off) <= P.k * G.slot_bytes;
        for (size_t j = gr.j0; j < gr.j1 && mirror; j++)
            mirror = P.mode[j] == kPlain && (j == gr.j0 || jobs[j].dst_off == jobs[j - 1].dst_off + jobs[j - 1].n);
        uint8_t* hs = G.pinned + slot_off(gr.j0);
        size_t wire_extent = 0;
        for (size_t j = gr.j0; j < gr.j1 && q.ok(); j++) {
            const Job& job = jobs[j];
            if (P.mode[j] == kHole) {
                q.ce = cudaMemsetAsync(d_dst + job.dst_off, 0, static_cast<size_t>(job.n), gr.cs);  // block_reader_hole.rs:69-79
                continue;
            }
            uint8_t* at = mirror ? hs + static_cast<size_t>(job.dst_off - first.dst_off) : G.pinned + slot_off(j);
            size_t wire = 0;
            CV_RETURN_IF_ERR(fetch(j, at, &wire));
            if (P.mode[j] == kFramed) {
                wire_extent = static_cast<size_t>(at - hs) + wire;
            } else {
                q.add(d_dst + job.dst_off, at, wire);
                if (!mirror) q.flush();
            }
        }
        if (wire_extent) q.add(G.d_stage + slot_off(gr.j0), hs, wire_extent);
        return Err::ok();
    }

    // ---- The tables.  off/len/expect/skip of every job, with the [f0, f1) window of the CRCs that are summed and the count of those
    // compared, and the scatter's tables go up in one copy; the result words are zeroed; a verbatim call's stream descriptors are
    // written here and uploaded per batch by the verifier, once the request ids are known.  The host image is pinned, owned by the
    // context, and rewritten only after the previous call's results were harvested (its uploads have long executed by then).
    Err write_tables() {
        const B200Conf& bc = r.ctx_->conf.b200;
        const TableLayout& tl = P.tl;
        const size_t J = jobs.size();
        CV_RETURN_IF_ERR(G.ensure_tables(tl.bytes, 4 * tl.res_words()));
        uint8_t* T = G.d_tables;
        uint8_t* h = G.h_tables;
        f0 = J, f1 = 0, n_compared = 0;
        for (size_t j = 0; j < J; j++) {
            const LocatedBlock& lb = *jobs[j].lb;
            tl.off(h)[j] = static_cast<uint64_t>(jobs[j].dst_off);
            tl.len(h)[j] = static_cast<uint64_t>(jobs[j].n);
            tl.expect(h)[j] = bc.verify_poly ? lb.crc32c : lb.crc32;
            tl.skip(h)[j] = !(jobs[j].full && lb.has_crc && P.mode[j] != kHole);
            if (!tl.skip(h)[j]) {
                f0 = std::min(f0, j), f1 = std::max(f1, j + 1);
                n_compared++;
            }
        }
        if (f0 >= f1) f0 = f1 = 0;
        // every whole block the manifest holds a CRC for is compared; holes, partial ranges and blocks without a manifest CRC are
        // masked out one by one (their CRCs are still computed, and summed when they lie inside [f0,f1))
        compare = bc.verify && n_compared > 0;
        if (scatter) scatter->write(tl.scatter(h));  // the scatter's tables ride in the same pinned image and the same copy
        CU_TRY(cudaMemcpyAsync(T, h, tl.o_crc, cudaMemcpyHostToDevice, G.vstream));
        CU_TRY(cudaMemsetAsync(tl.crc(T), 0, 4 * tl.res_words(), G.vstream));
        CvStreamDesc* sd = tl.streams(h);
        if (P.any_verbatim) {
            for (size_t j = 0; j < J; j++) {
                CvStreamDesc& d = sd[j];
                memset(&d, 0, sizeof(d));
                d.wire_off = slot_off(j), d.dst_off = tl.off(h)[j];
                d.block_len = P.mode[j] == kFramed ? static_cast<uint64_t>(P.wire_payload[j]) : 0;
                d.tail_clip = P.mode[j] == kFramed ? static_cast<uint32_t>(P.wire_payload[j] - jobs[j].n) : 0;
                d.chunk_size = static_cast<uint32_t>(P.chunk), d.first_seq_id = 1, d.block = static_cast<uint32_t>(j % P.B);
                d.first_frame = P.first_frame[j], d.code = kCodeReadBlock, d.status = 0x03;
            }
        }
        return Err::ok();
    }

    // ---- The verifier: this thread walks the copy groups in order, `vgroups` at a time, and fails the call on a launch error
    void verify_batches() {
        const B200Conf& bc = r.ctx_->conf.b200;
        const int poly = bc.verify_poly ? 1 : 0;
        const TableLayout& tl = P.tl;
        const size_t J = jobs.size();
        uint8_t* T = G.d_tables;
        const uint64_t* h_len = tl.len(G.h_tables);
        CvStreamDesc* sd = tl.streams(G.h_tables);
        uint32_t* d_crc = tl.crc(T);
        Err verr;
        for (size_t v0 = 0; v0 < P.NG && !verr; v0 += P.vgroups) {
            const size_t v1 = std::min(P.NG, v0 + P.vgroups);
            if (!await_copies(v0, v1)) break;
            const size_t g0 = v0 * P.k, g1 = std::min(J, v1 * P.k);
            uint64_t gbytes = 0;
            bool gframed = false;
            for (size_t g = v0; g < v1; g++) gframed |= P.group_verbatim[g] != 0;
            for (size_t j = g0; j < g1; j++) gbytes += h_len[j];
            if (!gframed && bc.verify) {  // K1 over the landed bytes
                int rc = cvk_crc_blocks(d_dst, tl.off(T) + g0, tl.len(T) + g0, static_cast<uint32_t>(g1 - g0), poly, gbytes, d_crc + g0, G.vstream);
                if (rc) verr = Err::io(str_printf("cvk_crc_blocks: %s", cudaGetErrorString(cudaError_t(rc))));
            }
            if (gframed) {
                // patch the request ids (known only after the fetch), expand this batch's stream descriptors, run K2
                for (size_t j = g0; j < g1; j++) sd[j].req_id = req_ids[j];
                cudaError_t ce = cudaMemcpyAsync(tl.streams(T) + g0, &sd[g0], sizeof(CvStreamDesc) * (g1 - g0), cudaMemcpyHostToDevice, G.vstream);
                const uint32_t fr0 = P.first_frame[g0], nfr = P.first_frame[g1] - fr0;
                int rc = ce != cudaSuccess ? int(ce) : 0;
                if (!rc) rc = cvk_expand_streams(tl.streams(T) + g0, static_cast<uint32_t>(g1 - g0), tl.fdesc(T), P.first_frame[J], G.vstream);
                if (!rc && nfr)
                    rc = cvk_unpack_frames(G.d_stage, tl.fdesc(T) + fr0, nfr, static_cast<uint32_t>(g1 - g0), d_dst, poly, gbytes,
                                           bc.verify ? d_crc + g0 : nullptr, tl.ferr(d_crc) + fr0, G.vstream);
                if (rc) verr = Err::io(str_printf("cvk_unpack_frames: %s", cudaGetErrorString(cudaError_t(rc))));
                release_verbatim(v0, v1);
            }
        }
        if (verr) fail(verr);
    }

    // ---- The finish: compare the CRCs with the manifest, scatter, copy the result words back, order the caller's stream after it all
    Err finish(cudaStream_t caller) {
        const TableLayout& tl = P.tl;
        uint8_t* T = G.d_tables;
        uint32_t* d_crc = tl.crc(T);
        if (compare)
            CVK_TRY(cvk_verify_crcs_masked(d_crc + f0, tl.expect(T) + f0, tl.skip(T) + f0, static_cast<uint32_t>(f1 - f0), tl.nbad(d_crc), nullptr, G.vstream));
        if (scatter)  // every copy group was waited for and CRC'd on vstream by now: deliver the landed bytes to their destinations
            CV_RETURN_IF_ERR(scatter->launch(d_dst, tl.scatter(T), G.vstream));
        CU_TRY(cudaMemcpyAsync(G.h_result, d_crc, 4 * tl.res_words(), cudaMemcpyDeviceToHost, G.vstream));
        CU_TRY(cudaEventRecord(G.done_ev, G.vstream));
        CU_TRY(cudaStreamWaitEvent(caller, G.done_ev, 0));
        return Err::ok();
    }

    void add_stats(uint64_t launches0, double t_start) {
        GpuReadStats& st = r.stats_;
        const uint64_t* h_len = P.tl.len(G.h_tables);
        for (size_t j = 0; j < jobs.size(); j++) st.bytes += h_len[j];
        st.blocks += jobs.size();
        st.kernel_launches += cvk_launch_count() - launches0;
        for (int t = 0; t < P.T_threads; t++) st.fetch_sec += fetch_sec[static_cast<size_t>(t)], st.h2d_bytes += h2d[static_cast<size_t>(t)];
        st.wall_sec += now_sec() - t_start;
        st.reg_hits = G.reg.hits.load(), st.reg_misses = G.reg.misses.load();
        st.reg_rejected = G.reg.rejected.load(), st.reg_bytes = G.reg.bytes();
        st.ring_alloc_sec = G.ring_alloc_sec;
        st.gds_bytes += gds_bytes.load();
    }
};

Err GpuFsReader::run_jobs(const std::vector<Job>& jobs, uint8_t* d_dst, void* user_stream, const Scatter* scatter) {
    if (jobs.empty()) return Err::ok();
    const double t_start = now_sec();
    GpuIngest& G = *ing_;
    struct InFlight {
        std::atomic<int>& n;
        explicit InFlight(std::atomic<int>& c) : n(c) { n.fetch_add(1, std::memory_order_acq_rel); }
        ~InFlight() { n.fetch_sub(1, std::memory_order_acq_rel); }
    } in_flight(G.reads_in_flight);
    std::lock_guard<std::mutex> call_lock(G.mu);
    CU_TRY(cudaSetDevice(G.device));
    CV_RETURN_IF_ERR(check_device_dst(d_dst, G.device));
    if (G.pending_owner && G.pending_owner != this) CV_RETURN_IF_ERR(G.pending_owner->harvest());  // shared tables
    CV_RETURN_IF_ERR(harvest());
    // everything this call writes into d_dst is ordered after what the caller's stream had queued at entry (a buffer fresh from
    // a stream-ordered allocator, kernels still reading it): the copy streams and the verify stream wait for that point
    CU_TRY(cudaEventRecord(G.entry_ev, static_cast<cudaStream_t>(user_stream)));
    for (auto cs : G.copy_streams) CU_TRY(cudaStreamWaitEvent(cs, G.entry_ev, 0));
    CU_TRY(cudaStreamWaitEvent(G.vstream, G.entry_ev, 0));
    const B200Conf& bc = ctx_->conf.b200;

    CallPlan P;
    CV_RETURN_IF_ERR(plan_call(jobs, scatter ? scatter->bytes() : 0, &P));
    Call c(*this, jobs, P, d_dst, scatter);
    if (!(bc.zero_copy && !P.call_framed)) CV_RETURN_IF_ERR(c.ensure_ring());
    CV_RETURN_IF_ERR(c.write_tables());

    // ---- fetch workers.  A verbatim (framed) group's slot is only released by the verifier below, so a single fetch worker running
    // inline on this thread would wait for itself once the groups outnumber the ring's super-slots: it gets its own thread then.
    std::vector<std::thread> threads;
    if (P.T_threads == 1 && (P.NG <= P.NS || !P.any_verbatim)) c.worker(0, false);  // small read (FUSE-shaped, C5): no thread spawn on the latency path
    else
        for (int t = 0; t < P.T_threads; t++) threads.emplace_back([&c, t] { c.worker(t, true); });

    const uint64_t launches0 = cvk_launch_count();
    c.verify_batches();
    for (auto& th : threads) th.join();
    if (c.err) {
        cudaStreamSynchronize(G.vstream);
        for (auto s : G.copy_streams) cudaStreamSynchronize(s);
        return c.err;
    }
    CV_RETURN_IF_ERR(c.finish(static_cast<cudaStream_t>(user_stream)));
    pending_.active = true, pending_.tl = P.tl;
    pending_.f0 = bc.verify ? c.f0 : 0, pending_.f1 = bc.verify ? c.f1 : 0, pending_.n_compared = c.compare ? c.n_compared : 0;
    G.pending_owner = this;
    c.add_stats(launches0, t_start);
    return Err::ok();
}

Err GpuFsReader::read_many(FsContext* ctx, const std::vector<std::string>& paths, const int64_t* dst_offs, void* d_dst, int64_t cap, void* stream,
                            uint64_t* sum_crc, uint32_t* n_bad, uint64_t* n_verified, int64_t* total_bytes) {
    std::unique_ptr<GpuFsReader> r(new GpuFsReader());
    r->ctx_ = ctx;
    Err e;
    r->ing_ = gpu_ingest_get(ctx, &e);
    if (e) return e;
    std::vector<Job> jobs;
    int64_t total = 0;
    for (size_t i = 0; i < paths.size(); i++) {
        std::shared_ptr<const FileBlocks> fb;
        CV_RETURN_IF_ERR(ctx->ns.get_block_locations(paths[i], &fb));
        r->held_files_.push_back(fb);
        if (dst_offs[i] < 0 || dst_offs[i] + fb->status.len > cap) return Err::common("destination too small for " + paths[i]);
        for (size_t b = 0; b < fb->block_locs.size(); b++) {
            const int64_t blen = fb->block_locs[b].block.len;
            if (blen > 0) jobs.push_back(Job{&fb->block_locs[b], 0, blen, dst_offs[i] + fb->starts[b], true});
        }
        total += fb->status.len;
    }
    if (!r->held_files_.empty()) r->fbp_ = r->held_files_[0];
    CV_RETURN_IF_ERR(r->run_jobs(jobs, static_cast<uint8_t*>(d_dst), stream));
    if (total_bytes) *total_bytes = total;
    return r->verify(sum_crc, n_bad, n_verified);
}

// Upper bound of the boundary-block staging of a vectored read, besides "no more blocks than the pinned ring has slots".
static const int64_t kReadvStageBytes = 256 << 20;

Err GpuFsReader::readv_device(const ReadvRange* ranges, int32_t n_ranges, void* stream, int64_t* n) {
    *n = 0;
    const FileBlocks& fb = *fbp_;
    std::vector<ReadvBlock> blocks;
    std::vector<ReadvSpan> spans;
    CV_RETURN_IF_ERR(plan_readv(fb, ranges, n_ranges, &blocks, &spans));
    GpuIngest& G = *ing_;
    CU_TRY(cudaSetDevice(G.device));
    int64_t total = 0;
    uintptr_t lo = UINTPTR_MAX;
    for (int32_t i = 0; i < n_ranges; i++) {
        const ReadvRange& r = ranges[i];
        if (r.row_len == 0 || r.rows == 0) continue;
        CV_RETURN_IF_ERR(check_device_dst(r.dst, G.device).ctx(str_printf("range %d", i)));
        const int64_t dst_row = dst_row_len(r);
        CV_RETURN_IF_ERR(check_device_dst(r.dst + (r.rows - 1) * r.dst_pitch + dst_row - 1, G.device).ctx(str_printf("range %d (last byte)", i)));
        if (r.scaled()) {  // the scale buffer too: its first and last byte (check_scale bounded its size)
            const uint8_t* sp = static_cast<const uint8_t*>(r.scale.ptr);
            CV_RETURN_IF_ERR(check_device_dst(sp, G.device).ctx(str_printf("range %d scale", i)));
            CV_RETURN_IF_ERR(check_device_dst(sp + r.scale.rows * r.scale.cols * dtype_size(r.scale.dtype) - 1, G.device)
                                 .ctx(str_printf("range %d scale (last byte)", i)));
        }
        lo = std::min(lo, reinterpret_cast<uintptr_t>(r.dst));
        total += r.rows * dst_row;
    }
    if (blocks.empty()) return Err::ok();
    std::vector<size_t> boundary;
    int64_t stage_block = 0;
    for (size_t b = 0; b < blocks.size(); b++)
        if (!blocks[b].direct) boundary.push_back(b), stage_block = std::max(stage_block, fb.block_locs[blocks[b].block].block.len);
    // One run_jobs call per round: the direct blocks and the first round of boundary blocks go in the first; later rounds reuse the
    // staging once the previous round's K3 has delivered it (run_jobs harvests the previous call on entry).
    std::lock_guard<std::mutex> lk(G.readv_mu);
    size_t per_round = 0;
    uint8_t* stage = nullptr;
    if (!boundary.empty()) {
        per_round = std::min(boundary.size(), static_cast<size_t>(std::max<int64_t>(1, std::min<int64_t>(G.nslots, kReadvStageBytes / stage_block))));
        CV_RETURN_IF_ERR(G.ensure_readv_stage(per_round * static_cast<size_t>(stage_block)));
        stage = G.d_readv_stage;
        lo = std::min(lo, reinterpret_cast<uintptr_t>(stage));
    }
    // every destination is addressed relative to the lowest one (or the staging): one base pointer, unsigned offsets
    uint8_t* base = reinterpret_cast<uint8_t*>(lo);
    auto rel = [lo](const uint8_t* p) { return static_cast<int64_t>(reinterpret_cast<uintptr_t>(p) - lo); };
    auto dst_of = [&](const ReadvSpan& s) { return rel(ranges[s.range].dst) + s.dst_off; };
    std::vector<Job> jobs;
    for (const ReadvBlock& b : blocks)
        if (b.direct) jobs.push_back(Job{&fb.block_locs[b.block], 0, spans[b.first_span].len, dst_of(spans[b.first_span]), true});
    size_t next = 0;
    do {
        Scatter sc(base);
        for (size_t slot = 0; slot < per_round && next < boundary.size(); slot++, next++) {
            const ReadvBlock& b = blocks[boundary[next]];
            const int64_t at = rel(stage + slot * static_cast<size_t>(stage_block));
            jobs.push_back(Job{&fb.block_locs[b.block], 0, fb.block_locs[b.block].block.len, at, true});
            for (size_t k = b.first_span; k < b.first_span + b.n_spans; k++) {
                const ReadvSpan& s = spans[k];
                sc.add(static_cast<uint64_t>(at + s.block_off), static_cast<uint64_t>(dst_of(s)), static_cast<uint64_t>(s.len), static_cast<uint64_t>(s.rows),
                       ranges[s.range], fb.starts[b.block] + s.block_off);
            }
        }
        CV_RETURN_IF_ERR(run_jobs(jobs, base, stream, &sc));
        jobs.clear();
    } while (next < boundary.size());
    *n = total;
    return Err::ok();
}

}  // namespace cv
