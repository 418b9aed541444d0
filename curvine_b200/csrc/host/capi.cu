// extern "C" surface declared in include/curvine_b200.h (upper boundary).  Never throws, never aborts:
// every failure becomes -(ErrorKind) plus a thread-local message (cv_last_error).
#include <cuda_runtime.h>
#include <nmmintrin.h>
#include <errno.h>
#include <fcntl.h>
#include <stdlib.h>
#include <unistd.h>

#include <fstream>
#include <thread>

#include "../../../include/curvine_b200.h"
#include "../crc_gf.h"
#include "client.h"
#include "gds.h"
#include "gpu_reader.h"
#include "numa.h"
#include "worker.h"
#include "writer.h"

using namespace cv;

static thread_local std::string g_last_error;

static int64_t fail(const Err& e) {
    g_last_error = e.msg;
    return e.libc_kind();
}
static int64_t ok() { return 0; }

#define API_TRY(expr)             \
    do {                          \
        Err e__ = (expr);         \
        if (e__) return fail(e__); \
    } while (0)
// every handle / required out-pointer is checked before it is touched: a NULL comes back as -(Common) with a message, never a crash
#define API_NEED(x)                                                          \
    do {                                                                     \
        if (!(x)) return fail(Err::common("null argument: " #x));           \
    } while (0)
#define API_GUARD_BEGIN try {
#define API_GUARD_END                                                     \
    }                                                                     \
    catch (const std::exception& ex) {                                    \
        return fail(Err::common(std::string("internal: ") + ex.what())); \
    }                                                                     \
    catch (...) {                                                         \
        return fail(Err::common("internal: unknown exception"));         \
    }

// The filesystem context is shared between the filesystem handle and every reader / writer opened from it, as in the reference
// (FsReader and FsWriter hold an Arc<FsContext>; closeFilesystem only drops the handle's reference: lib_filesystem.rs:25-40): a reader
// that outlives its filesystem handle stays valid, and the GPU ingest pipeline goes with the LAST holder.
static std::shared_ptr<FsContext> make_context(const ClusterConf& c) {
    return std::shared_ptr<FsContext>(new FsContext(c), [](FsContext* ctx) {
        gpu_ingest_release(ctx);
        delete ctx;
    });
}

struct cv_fs {
    std::shared_ptr<FsContext> ctx;
};

struct cv_reader {
    std::shared_ptr<FsContext> ctx;  // first member: destroyed after the readers below
    std::string path;
    std::unique_ptr<FsReader> host;
    std::unique_ptr<GpuFsReader> dev;
};

struct cv_writer {
    std::shared_ptr<FsContext> ctx;  // first member: destroyed after the writer below
    std::unique_ptr<FsWriter> w;
};

struct cv_worker {
    Worker w;
    std::string hostname;
};

static Err ensure_dev(cv_reader* r) {
    if (r->dev) return Err::ok();
    return GpuFsReader::open(r->ctx.get(), r->path, &r->dev);
}

// One ReadvRange per ABI range: a plain range is a strided range of one row, a cast range a strided range with dtypes, a scaled range
// a cast range with a scale.
static ReadvRange to_readv(const CvRange& s) { return ReadvRange{s.file_off, s.len, static_cast<uint8_t*>(s.d_dst)}; }

static ReadvRange to_readv(const CvStridedRange& s) {
    return ReadvRange{s.file_off, s.row_len, static_cast<uint8_t*>(s.d_dst), s.rows, s.file_pitch, s.dst_pitch};
}

static ReadvRange to_readv(const CvCastRange& s) {
    return ReadvRange{s.file_off, s.row_len, static_cast<uint8_t*>(s.d_dst), s.rows, s.file_pitch, s.dst_pitch, s.src_dtype, s.dst_dtype};
}

static ReadvRange to_readv(const CvScaledRange& s) {
    ReadvRange r = to_readv(s.cast);
    r.scale = ReadvScale{s.d_scale, s.scale_dtype, s.scale_rows, s.scale_cols, s.block_rows, s.block_cols, s.cols, s.first_elem};
    return r;
}

template <typename Range>
static std::vector<ReadvRange> to_readv(const Range* ranges, int32_t n) {
    std::vector<ReadvRange> out;
    for (int32_t i = 0; ranges && i < n; i++) out.push_back(to_readv(ranges[i]));
    return out;
}

template <typename Range>
static int64_t readv_device_body(cv_reader* r, const Range* ranges, int32_t n, cv_stream_t stream, int64_t* nbytes) {
    API_TRY(ensure_dev(r));
    const std::vector<ReadvRange> rs = to_readv(ranges, n);
    int64_t got = 0;
    API_TRY(r->dev->readv_device(rs.data(), n, stream, &got));
    *nbytes = got;
    return ok();
}

// The plan's spans into the caller's arrays (any of which may be NULL); `rows` only for the strided form.
template <typename Range>
static int64_t readv_plan_body(cv_reader* r, const Range* ranges, int32_t n, int64_t* block_index, int64_t* block_off, int64_t* len, int64_t* rows,
                               int32_t* range_index, int32_t* direct, int32_t cap, int32_t* n_spans, int64_t* n_blocks, int64_t* fetch_bytes) {
    const FileBlocks& fb = r->host->file_blocks();
    const std::vector<ReadvRange> rs = to_readv(ranges, n);
    std::vector<ReadvBlock> blocks;
    std::vector<ReadvSpan> spans;
    API_TRY(plan_readv(fb, rs.data(), n, &blocks, &spans));
    int64_t fetched = 0;
    size_t i = 0;
    for (const ReadvBlock& b : blocks) {
        fetched += fb.block_locs[b.block].block.len;
        for (size_t k = b.first_span; k < b.first_span + b.n_spans; k++, i++) {
            if (i >= static_cast<size_t>(std::max(cap, 0))) continue;
            if (block_index) block_index[i] = static_cast<int64_t>(b.block);
            if (block_off) block_off[i] = spans[k].block_off;
            if (len) len[i] = spans[k].len;
            if (rows) rows[i] = spans[k].rows;
            if (range_index) range_index[i] = spans[k].range;
            if (direct) direct[i] = b.direct ? 1 : 0;
        }
    }
    if (n_spans) *n_spans = static_cast<int32_t>(spans.size());
    if (n_blocks) *n_blocks = static_cast<int64_t>(blocks.size());
    if (fetch_bytes) *fetch_bytes = fetched;
    return ok();
}

extern "C" {

const char* cv_last_error(void) { return g_last_error.c_str(); }
void cv_free(void* p) { free(p); }

int64_t cv_fs_new_from_string(const char* conf_toml, cv_fs** out) {
    API_GUARD_BEGIN
    API_NEED(out);
    ClusterConf c;
    API_TRY(ClusterConf::from_string(conf_toml ? conf_toml : "", &c));
    std::unique_ptr<cv_fs> fs(new cv_fs());
    fs->ctx = make_context(c);
    if (!c.namespace_manifest.empty()) API_TRY(fs->ctx->ns.load(c.namespace_manifest));
    *out = fs.release();
    return ok();
    API_GUARD_END
}

int64_t cv_fs_new(const char* conf_path, cv_fs** out) {
    API_GUARD_BEGIN
    API_NEED(out);
    ClusterConf c;
    // no path given: $CURVINE_CONF_FILE, the fallback the reference's entry points use (ClusterConf::ENV_CONF_FILE, cluster_conf.rs:76; curvine-cli/src/main.rs:62)
    const char* env_path = getenv("CURVINE_CONF_FILE");
    API_TRY(ClusterConf::from_file(conf_path && *conf_path ? conf_path : (env_path ? env_path : ""), &c));
    std::unique_ptr<cv_fs> fs(new cv_fs());
    fs->ctx = make_context(c);
    if (!c.namespace_manifest.empty()) API_TRY(fs->ctx->ns.load(c.namespace_manifest));
    *out = fs.release();
    return ok();
    API_GUARD_END
}

int64_t cv_fs_load_namespace(cv_fs* fs, const char* manifest_path) {
    API_GUARD_BEGIN
    API_NEED(fs);
    API_NEED(manifest_path);
    API_TRY(fs->ctx->ns.load(manifest_path));
    return ok();
    API_GUARD_END
}

int64_t cv_fs_load_namespace_string(cv_fs* fs, const char* text) {
    API_GUARD_BEGIN
    API_NEED(fs);
    API_NEED(text);
    API_TRY(fs->ctx->ns.load_string(text));
    return ok();
    API_GUARD_END
}

int64_t cv_fs_close(cv_fs* fs) {
    API_GUARD_BEGIN
    if (!fs) return ok();
    delete fs;  // drops the handle's reference; open readers / writers keep the context (and its GPU pipeline) until they are closed
    return ok();
    API_GUARD_END
}

int64_t cv_fs_wait_registered(cv_fs* fs) {
    API_GUARD_BEGIN
    API_NEED(fs);
    gpu_ingest_wait_registered(fs->ctx.get());
    return ok();
    API_GUARD_END
}

int64_t cv_fs_preregister(cv_fs* fs) {
    API_GUARD_BEGIN
    API_NEED(fs);
    API_TRY(gpu_ingest_preregister(fs->ctx.get()));
    return ok();
    API_GUARD_END
}

int64_t cv_fs_arena_stats(cv_fs* fs, uint64_t out[5]) {
    API_NEED(fs);
    API_NEED(out);
    gpu_ingest_arena_stats(fs->ctx.get(), out);
    return ok();
}

int64_t cv_fs_metrics(cv_fs* fs, int64_t out[2]) {
    API_NEED(fs);
    API_NEED(out);
    out[0] = fs->ctx->read_bytes.load(), out[1] = fs->ctx->read_time_us.load();
    return ok();
}

int64_t cv_fs_pool_stats(cv_fs* fs, int64_t out[3]) {
    API_NEED(fs);
    API_NEED(out);
    fs->ctx->pool_stats(out);
    return ok();
}

int64_t cv_open(cv_fs* fs, const char* path, cv_reader** out, int64_t* len) {
    API_GUARD_BEGIN
    API_NEED(fs);
    API_NEED(path);
    API_NEED(out);
    std::unique_ptr<cv_reader> r(new cv_reader());
    r->ctx = fs->ctx, r->path = path;
    API_TRY(FsReader::open(fs->ctx.get(), path, &r->host));
    if (len) *len = r->host->len();
    *out = r.release();
    return ok();
    API_GUARD_END
}

int64_t cv_read(cv_reader* r, const uint8_t** ptr, int64_t* len) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_NEED(ptr);
    API_NEED(len);
    API_TRY(r->host->read_chunk(ptr, len, -1));
    return ok();
    API_GUARD_END
}

int64_t cv_read_buf(cv_reader* r, uint8_t* buf, int64_t cap, int64_t* n) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_NEED(n);
    API_TRY(r->host->read(buf, cap, n));
    return ok();
    API_GUARD_END
}

int64_t cv_read_full(cv_reader* r, uint8_t* buf, int64_t cap, int64_t* n) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_NEED(n);
    API_TRY(r->host->read_full(buf, cap, n));
    return ok();
    API_GUARD_END
}

int64_t cv_fuse_read(cv_reader* r, int64_t pos, int64_t len, uint8_t* buf, int64_t* n, int64_t* seg_lens, int32_t max_segs,
                     int32_t* n_segs) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_TRY(r->host->seek(pos));
    int64_t remaining = len, off = 0;
    int32_t segs = 0;
    while (remaining > 0) {
        const uint8_t* p;
        int64_t got;
        API_TRY(r->host->read_chunk(&p, &got, remaining));
        if (got == 0) break;
        memcpy(buf + off, p, static_cast<size_t>(got));
        if (seg_lens && segs < max_segs) seg_lens[segs] = got;
        segs++, off += got, remaining -= got;
    }
    if (n) *n = off;
    if (n_segs) *n_segs = segs;
    return ok();
    API_GUARD_END
}

int64_t cv_seek(cv_reader* r, int64_t pos) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_TRY(r->host->seek(pos));
    return ok();
    API_GUARD_END
}

int64_t cv_pos(cv_reader* r) { return r ? r->host->pos() : -int64_t(kCommon); }
int64_t cv_len(cv_reader* r) { return r ? r->host->len() : -int64_t(kCommon); }
int64_t cv_chunk_size(cv_reader* r) { return r ? r->host->chunk_size() : -int64_t(kCommon); }

int64_t cv_close_reader(cv_reader* r) {
    API_GUARD_BEGIN
    if (!r) return ok();
    Err e = r->host ? r->host->complete() : Err::ok();
    if (r->dev) {
        Err e2 = r->dev->complete();
        if (!e && e2) e = e2;
    }
    delete r;
    if (e) return fail(e);
    return ok();
    API_GUARD_END
}

int64_t cv_read_device(cv_reader* r, void* d_dst, int64_t cap, cv_stream_t stream, int64_t* nbytes) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_NEED(nbytes);
    API_TRY(ensure_dev(r));
    API_TRY(r->dev->seek(r->host->pos()));
    int64_t n = 0;
    API_TRY(r->dev->read_device(d_dst, cap, stream, &n));
    API_TRY(r->host->seek(r->dev->pos()));
    if (nbytes) *nbytes = n;
    return ok();
    API_GUARD_END
}

int64_t cv_read_device_sharded(cv_reader* r, int32_t rank, int32_t world, void* d_dst, int64_t cap, cv_stream_t stream,
                               int64_t* nbytes) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_NEED(nbytes);
    API_TRY(ensure_dev(r));
    int64_t n = 0;
    API_TRY(r->dev->read_device_sharded(rank, world, d_dst, cap, stream, &n));
    if (nbytes) *nbytes = n;
    return ok();
    API_GUARD_END
}

int64_t cv_read_many_device(cv_fs* fs, const char* const* paths, int32_t n, void* d_dst, const int64_t* dst_offs, int64_t cap, cv_stream_t stream,
                            uint64_t* sum_crc, uint32_t* n_bad, uint64_t* n_verified, int64_t* total_bytes) {
    API_GUARD_BEGIN
    API_NEED(fs);
    API_NEED(paths);
    API_NEED(dst_offs);
    std::vector<std::string> ps;
    for (int32_t i = 0; i < n; i++) ps.emplace_back(paths[i]);
    uint64_t s = 0, v = 0;
    uint32_t b = 0;
    int64_t t = 0;
    API_TRY(GpuFsReader::read_many(fs->ctx.get(), ps, dst_offs, d_dst, cap, stream, &s, &b, &v, &t));
    if (sum_crc) *sum_crc = s;
    if (n_bad) *n_bad = b;
    if (n_verified) *n_verified = v;
    if (total_bytes) *total_bytes = t;
    return ok();
    API_GUARD_END
}

int64_t cv_shard_plan(cv_reader* r, int32_t rank, int32_t world, int64_t* block_index, int64_t* file_off, int64_t* len, int64_t* dst_off,
                      int32_t cap, int32_t* n, int64_t* total_bytes) {
    API_GUARD_BEGIN
    API_NEED(r);
    std::vector<ShardJob> plan;
    int64_t total = 0;
    API_TRY(plan_shard(r->host->file_blocks(), rank, world, -1, &plan, &total));
    if (n) *n = static_cast<int32_t>(plan.size());
    if (total_bytes) *total_bytes = total;
    for (size_t i = 0; i < plan.size() && static_cast<int32_t>(i) < cap; i++) {
        if (block_index) block_index[i] = static_cast<int64_t>(plan[i].block);
        if (file_off) file_off[i] = plan[i].file_off;
        if (len) len[i] = plan[i].len;
        if (dst_off) dst_off[i] = plan[i].dst_off;
    }
    return ok();
    API_GUARD_END
}

int64_t cv_readv_device(cv_reader* r, const CvRange* ranges, int32_t n, cv_stream_t stream, int64_t* nbytes) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_NEED(nbytes);
    if (n > 0) API_NEED(ranges);
    return readv_device_body(r, ranges, n, stream, nbytes);
    API_GUARD_END
}

int64_t cv_readv_plan(cv_reader* r, const CvRange* ranges, int32_t n, int64_t* block_index, int64_t* block_off, int64_t* len, int32_t* range_index,
                      int32_t* direct, int32_t cap, int32_t* n_spans, int64_t* n_blocks, int64_t* fetch_bytes) {
    API_GUARD_BEGIN
    API_NEED(r);
    if (n > 0) API_NEED(ranges);
    return readv_plan_body(r, ranges, n, block_index, block_off, len, nullptr, range_index, direct, cap, n_spans, n_blocks, fetch_bytes);
    API_GUARD_END
}

int64_t cv_readv_strided_device(cv_reader* r, const CvStridedRange* ranges, int32_t n, cv_stream_t stream, int64_t* nbytes) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_NEED(nbytes);
    if (n > 0) API_NEED(ranges);
    return readv_device_body(r, ranges, n, stream, nbytes);
    API_GUARD_END
}

int64_t cv_readv_strided_plan(cv_reader* r, const CvStridedRange* ranges, int32_t n, int64_t* block_index, int64_t* block_off, int64_t* len, int64_t* rows,
                              int32_t* range_index, int32_t* direct, int32_t cap, int32_t* n_spans, int64_t* n_blocks, int64_t* fetch_bytes) {
    API_GUARD_BEGIN
    API_NEED(r);
    if (n > 0) API_NEED(ranges);
    return readv_plan_body(r, ranges, n, block_index, block_off, len, rows, range_index, direct, cap, n_spans, n_blocks, fetch_bytes);
    API_GUARD_END
}

int64_t cv_readv_cast_device(cv_reader* r, const CvCastRange* ranges, int32_t n, cv_stream_t stream, int64_t* nbytes) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_NEED(nbytes);
    if (n > 0) API_NEED(ranges);
    return readv_device_body(r, ranges, n, stream, nbytes);
    API_GUARD_END
}

int64_t cv_readv_scaled_device(cv_reader* r, const CvScaledRange* ranges, int32_t n, cv_stream_t stream, int64_t* nbytes) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_NEED(nbytes);
    if (n > 0) API_NEED(ranges);
    return readv_device_body(r, ranges, n, stream, nbytes);
    API_GUARD_END
}

int64_t cv_readv_cast_plan(cv_reader* r, const CvCastRange* ranges, int32_t n, int64_t* block_index, int64_t* block_off, int64_t* len, int64_t* rows,
                           int32_t* range_index, int32_t* direct, int32_t cap, int32_t* n_spans, int64_t* n_blocks, int64_t* fetch_bytes) {
    API_GUARD_BEGIN
    API_NEED(r);
    if (n > 0) API_NEED(ranges);
    return readv_plan_body(r, ranges, n, block_index, block_off, len, rows, range_index, direct, cap, n_spans, n_blocks, fetch_bytes);
    API_GUARD_END
}

int64_t cv_fuse_read_device(cv_reader* r, int64_t pos, int64_t len, void* d_scratch, void* d_page_base, const uint64_t* page_offsets,
                            int32_t n_pages, int64_t page_size, cv_stream_t stream, int64_t* nbytes) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_NEED(page_offsets);
    API_TRY(ensure_dev(r));
    API_TRY(r->host->seek(pos));
    API_TRY(r->dev->seek(pos));
    int64_t n = 0;
    // ResponseData::as_iovec analogue on the device: the bytes land in the scratch, are CRC'd, and go to the reply's page buffers
    // in the same launch train (segment table in the reader's pinned staging: no allocation, no synchronisation here)
    API_TRY(r->dev->fuse_read_device(len, d_scratch, d_page_base, page_offsets, n_pages, page_size, stream, &n));
    API_TRY(r->host->seek(r->dev->pos()));
    if (nbytes) *nbytes = n;
    return ok();
    API_GUARD_END
}

// open -> fuse_read(0, len) -> verify -> close of ONE file in one call: what a FUSE daemon does for a small file
// (reader.rs:101-124 behind FileSystem::open / Reader::complete), without four trips through the binding
int64_t cv_fuse_read_file_device(cv_fs* fs, const char* path, int64_t len, void* d_scratch, void* d_page_base, const uint64_t* page_offsets, int32_t n_pages,
                                 int64_t page_size, cv_stream_t stream, int64_t* nbytes, uint32_t* n_bad) {
    API_GUARD_BEGIN
    API_NEED(fs);
    API_NEED(path);
    API_NEED(page_offsets);
    std::unique_ptr<GpuFsReader> dev;
    API_TRY(GpuFsReader::open(fs->ctx.get(), path, &dev));
    int64_t n = 0;
    API_TRY(dev->fuse_read_device(len, d_scratch, d_page_base, page_offsets, n_pages, page_size, stream, &n));
    uint64_t s = 0, v = 0;
    uint32_t b = 0;
    API_TRY(dev->verify(&s, &b, &v));
    if (nbytes) *nbytes = n;
    if (n_bad) *n_bad = b;
    return ok();
    API_GUARD_END
}

int64_t cv_verify(cv_reader* r, uint64_t* sum_crc, uint32_t* n_bad, uint64_t* n_verified) {
    API_GUARD_BEGIN
    API_NEED(r);
    API_NEED(sum_crc);
    API_NEED(n_bad);
    API_NEED(n_verified);
    uint64_t s = 0, v = 0;
    uint32_t b = 0;
    if (r->dev) API_TRY(r->dev->verify(&s, &b, &v));
    if (sum_crc) *sum_crc = s;
    if (n_bad) *n_bad = b;
    if (n_verified) *n_verified = v;
    return ok();
    API_GUARD_END
}

int64_t cv_device_stats(cv_reader* r, CvReadStats* out) {
    API_NEED(r);
    API_NEED(out);
    memset(out, 0, sizeof(*out));
    if (!r->dev) return ok();
    const GpuReadStats& s = r->dev->stats();
    out->bytes = s.bytes, out->blocks = s.blocks, out->verified = s.verified, out->h2d_bytes = s.h2d_bytes;
    out->kernel_launches = s.kernel_launches, out->fetch_sec = s.fetch_sec, out->wall_sec = s.wall_sec;
    out->reg_hits = s.reg_hits, out->reg_misses = s.reg_misses;
    out->ring_alloc_sec = s.ring_alloc_sec;
    out->reg_rejected = s.reg_rejected, out->reg_bytes = s.reg_bytes;
    out->gds_bytes = s.gds_bytes;
    return ok();
}

int64_t cv_gds_info(int64_t out[2]) {
    API_NEED(out);
    const GdsInfo& g = gds_info();
    out[0] = g.available, out[1] = 0;  // out[1]: reserved (cuFile's compatibility mode is never used)
    g_last_error = g.detail;
    const std::string why = gds_last_refusal();
    if (!why.empty()) g_last_error += "; first refusal: " + why;
    return ok();
}

// ------------------------------------------------------------------ write-side mirror (SURVEY.md 8f-1)

int64_t cv_writer_open(cv_fs* fs, const char* path, int64_t inode_id, int64_t block_size, int32_t storage_type, const char* worker_host,
                       int32_t worker_port, int64_t chunk_size, cv_writer** out) {
    API_GUARD_BEGIN
    API_NEED(fs);
    API_NEED(path);
    API_NEED(worker_host);
    API_NEED(out);
    WorkerAddress a;
    a.worker_id = 1, a.hostname = worker_host, a.ip_addr = "127.0.0.1", a.rpc_port = static_cast<uint32_t>(worker_port);
    if (a.hostname != "localhost") a.ip_addr = a.hostname;
    std::unique_ptr<cv_writer> w(new cv_writer());
    w->ctx = fs->ctx;
    API_TRY(FsWriter::create(fs->ctx.get(), path, inode_id, block_size, storage_type, a, chunk_size > 0 ? chunk_size : 128 * 1024, &w->w));
    *out = w.release();
    return ok();
    API_GUARD_END
}

int64_t cv_write(cv_writer* w, const uint8_t* buf, int64_t n) {
    API_GUARD_BEGIN
    API_NEED(w);
    API_TRY(w->w->write(buf, n));
    return ok();
    API_GUARD_END
}

int64_t cv_write_device(cv_writer* w, const void* d_src, int64_t n, cv_stream_t stream) {
    API_GUARD_BEGIN
    API_NEED(w);
    API_TRY(w->w->write_device(d_src, n, stream));
    return ok();
    API_GUARD_END
}

int64_t cv_writer_close(cv_writer* w, int32_t cancel, char** manifest_out) {
    API_GUARD_BEGIN
    API_NEED(w);
    if (!w) return ok();
    Err e = cancel ? w->w->cancel() : w->w->complete();
    if (!e && manifest_out) {
        const std::string text = w->w->manifest();
        *manifest_out = static_cast<char*>(malloc(text.size() + 1));
        memcpy(*manifest_out, text.c_str(), text.size() + 1);
    }
    delete w;
    if (e) return fail(e);
    return ok();
    API_GUARD_END
}

// ------------------------------------------------------------------ fixture: worker + synthetic files

int64_t cv_worker_start(const char* conf_toml, cv_worker** out, int32_t* port) {
    API_GUARD_BEGIN
    API_NEED(out);
    ClusterConf c;
    API_TRY(ClusterConf::from_string(conf_toml ? conf_toml : "", &c));
    std::unique_ptr<cv_worker> w(new cv_worker());
    w->hostname = c.worker_hostname;
    w->w.hbm().configure(c.worker_hbm_capacity, c.worker_hbm_promote_after, c.worker_hbm_device);
    ArenaOpts ao;
    ao.enable = c.worker_mem_arena, ao.seg_bytes = c.worker_arena_segment, ao.numa = c.worker_arena_numa, ao.reuse_delay_ms = c.worker_arena_reuse_delay_ms;
    API_TRY(w->w.start(c.worker_dirs, c.cluster_id, "", c.worker_port, c.worker_enable_send_file, ao));
    if (port) *port = w->w.port();
    *out = w.release();
    return ok();
    API_GUARD_END
}

int64_t cv_worker_stop(cv_worker* w) {
    API_GUARD_BEGIN
    if (!w) return ok();
    w->w.stop();
    delete w;
    return ok();
    API_GUARD_END
}

int64_t cv_worker_hbm_load(cv_worker* w, int64_t block_id, int32_t device) {
    API_GUARD_BEGIN
    API_NEED(w);
    BlockMeta m;
    API_TRY(w->w.store().get_block(block_id, &m));
    std::ifstream f(m.path, std::ios::binary);
    if (!f) return fail(Err::io("open " + m.path));
    std::vector<char> buf(static_cast<size_t>(m.len));
    f.read(buf.data(), static_cast<std::streamsize>(buf.size()));
    if (f.gcount() != static_cast<std::streamsize>(buf.size())) return fail(Err::io("short read of " + m.path));
    API_TRY(w->w.hbm().load(block_id, buf.data(), m.len, device));
    return ok();
    API_GUARD_END
}

int64_t cv_worker_hbm_drain(cv_worker* w) {
    API_GUARD_BEGIN
    API_NEED(w);
    w->w.hbm().drain();
    return ok();
    API_GUARD_END
}

int64_t cv_worker_hbm_stats(cv_worker* w, int64_t out[3]) {
    API_NEED(w);
    API_NEED(out);
    WorkerMetrics& m = w->w.metrics();
    out[0] = static_cast<int64_t>(w->w.hbm().size()), out[1] = m.read_blocks_hbm, out[2] = m.hbm_packed_bytes;
    return ok();
}

int64_t cv_worker_hbm_tier(cv_worker* w, int64_t out[6]) {
    API_NEED(w);
    API_NEED(out);
    w->w.hbm().stats(out);
    return ok();
}

int64_t cv_worker_metrics(cv_worker* w, int64_t out[6]) {
    API_NEED(w);
    API_NEED(out);
    WorkerMetrics& m = w->w.metrics();
    out[0] = m.read_bytes, out[1] = m.read_time_us, out[2] = m.read_count, out[3] = m.read_blocks_local, out[4] = m.read_blocks_remote;
    out[5] = static_cast<int64_t>(w->w.store().num_blocks());
    return ok();
}

int64_t cv_synth_delete_file(cv_worker* w, int64_t inode_id, int64_t n_blocks) {
    API_GUARD_BEGIN
    API_NEED(w);
    for (int64_t b = 0; b < n_blocks; b++) {
        int64_t id = 0;
        API_TRY(create_block_id(inode_id, b, &id));
        w->w.hbm().evict(id);
        w->w.store().remove_block(id);
    }
    return ok();
    API_GUARD_END
}

int64_t cv_worker_arena_stats(cv_worker* w, int64_t out[5]) {
    API_NEED(w);
    API_NEED(out);
    memset(out, 0, 5 * sizeof(int64_t));
    double sec = 0;
    for (const auto& d : w->w.store().dirs())
        if (d.arena) {
            out[0]++, out[1] += static_cast<int64_t>(d.arena->num_segments()), out[2] = d.arena->seg_bytes(), out[3] += d.arena->used_bytes();
            sec += d.arena->populate_sec;
        }
    out[4] = static_cast<int64_t>(sec * 1e6);
    return ok();
}

static inline uint64_t rotl64(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }

void cv_synth_block(uint64_t file_id, uint64_t block_index, uint8_t* out, size_t len) {
    uint64_t x = 0xC0FFEEB200ull ^ (file_id << 32) ^ block_index, s[4];
    for (int i = 0; i < 4; i++) {
        x += 0x9E3779B97F4A7C15ull;
        uint64_t z = x;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        s[i] = z ^ (z >> 31);
    }
    size_t pos = 0;
    while (pos < len) {
        const uint64_t r = rotl64(s[1] * 5, 7) * 9, t = s[1] << 17;
        s[2] ^= s[0], s[3] ^= s[1], s[1] ^= s[2], s[0] ^= s[3], s[2] ^= t, s[3] = rotl64(s[3], 45);
        const size_t n = len - pos < 8 ? len - pos : 8;
        memcpy(out + pos, &r, n);
        pos += n;
    }
}

uint32_t cv_host_crc(int poly, const uint8_t* buf, size_t len) {
    if (poly == 1) {  // CRC-32C: SSE4.2 crc32 instruction
        uint64_t r = 0xffffffffu;
        while (len && (reinterpret_cast<uintptr_t>(buf) & 7)) r = _mm_crc32_u8(static_cast<uint32_t>(r), *buf++), len--;
        while (len >= 8) {
            uint64_t w;
            memcpy(&w, buf, 8);
            r = _mm_crc32_u64(r, w);
            buf += 8, len -= 8;
        }
        while (len--) r = _mm_crc32_u8(static_cast<uint32_t>(r), *buf++);
        return ~static_cast<uint32_t>(r);
    }
    static uint32_t T[8][256];
    static std::once_flag once;
    std::call_once(once, [] {
        for (uint32_t i = 0; i < 256; i++) {
            uint32_t r = i;
            for (int k = 0; k < 8; k++) r = gf_mulx(r, kPolyIeee);
            T[0][i] = r;
        }
        for (uint32_t i = 0; i < 256; i++)
            for (int s = 1; s < 8; s++) T[s][i] = (T[s - 1][i] >> 8) ^ T[0][T[s - 1][i] & 0xff];
    });
    uint32_t r = 0xffffffffu;
    while (len >= 8) {
        uint64_t w;
        memcpy(&w, buf, 8);
        const uint32_t lo = static_cast<uint32_t>(w) ^ r, hi = static_cast<uint32_t>(w >> 32);
        r = T[7][lo & 0xff] ^ T[6][(lo >> 8) & 0xff] ^ T[5][(lo >> 16) & 0xff] ^ T[4][lo >> 24] ^ T[3][hi & 0xff] ^ T[2][(hi >> 8) & 0xff] ^
            T[1][(hi >> 16) & 0xff] ^ T[0][hi >> 24];
        buf += 8, len -= 8;
    }
    while (len--) r = T[0][(r ^ *buf++) & 0xff] ^ (r >> 8);
    return ~r;
}

// CPUs of the NUMA node each CUDA device hangs off (empty when unknown)
static std::vector<std::vector<int>> gpu_node_cpus() {
    std::vector<std::vector<int>> out;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return out;
    }
    for (int d = 0; d < n; d++) out.push_back(node_cpus(gpu_numa_node(d)));
    return out;
}

// NUMA node of the PCIe root the device hangs off (-1 unknown): where its mem arena and fetch threads should live
int64_t cv_gpu_numa_node(int32_t device) { return gpu_numa_node(device); }

static int g_synth_shard_world = 0;

// NUMA-aware mem-tier placement for round-robin shards: with shard_world = G, block b of files created afterwards is
// first-touched (tmpfs pages allocated) on the NUMA node of GPU b % G, so every GPU later DMAs from local memory.
int64_t cv_synth_set_shard_world(int32_t shard_world) {
    g_synth_shard_world = shard_world;
    return ok();
}

int64_t cv_synth_create_file(cv_worker* w, const char* path, int64_t inode_id, int64_t len, int64_t block_size, int32_t storage_type,
                             int32_t mode, int32_t hole_every, int32_t threads, const char* worker_hostname, char** manifest_out) {
    API_GUARD_BEGIN
    API_NEED(w);
    API_NEED(path);
    API_NEED(manifest_out);
    std::vector<std::vector<int>> node_cpus;
    if (g_synth_shard_world >= 1) node_cpus = gpu_node_cpus();
    if (block_size <= 0 || len < 0) return fail(Err(kInvalidFileSize, "bad file or block size"));
    const int64_t nb = (len + block_size - 1) / block_size;
    FileBlocks fb;
    fb.status.id = inode_id, fb.status.path = path, fb.status.len = len, fb.status.block_size = block_size, fb.status.mtime = 0;
    fb.block_locs.resize(static_cast<size_t>(nb));
    WorkerAddress addr;
    addr.worker_id = 1, addr.hostname = worker_hostname && *worker_hostname ? worker_hostname : w->hostname, addr.ip_addr = "127.0.0.1";
    addr.rpc_port = static_cast<uint32_t>(w->w.port());
    std::string az;
    if (mode == 1) {  // curvine-bench style content: one a-z buffer repeated (bench_action.rs:100-102)
        az.resize(static_cast<size_t>(std::min<int64_t>(block_size, 128 * 1024)));
        uint64_t x = 42;
        for (auto& c : az) {
            x += 0x9E3779B97F4A7C15ull;
            uint64_t z = x;
            z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull, z = (z ^ (z >> 27)) * 0x94D049BB133111EBull, z ^= z >> 31;
            c = static_cast<char>('a' + z % 26);
        }
    }
    // Places first, in block order on this thread: in an arena dir consecutive blocks (of one placement class) get back-to-back
    // extents, so a reader later moves a whole copy group with one DMA.  The bytes are then produced in parallel -- straight
    // into the extent for arena dirs, through a buffer + write(2) for file dirs.
    std::vector<BlockWriteTarget> targets(static_cast<size_t>(nb));
    std::vector<uint8_t> is_hole(static_cast<size_t>(nb), 0);
    for (int64_t b = 0; b < nb; b++) {
        LocatedBlock& lb = fb.block_locs[static_cast<size_t>(b)];
        int64_t id = 0;
        API_TRY(create_block_id(inode_id, b, &id));
        const int64_t blen = std::min(block_size, len - b * block_size);
        lb.block.id = id, lb.block.len = blen, lb.block.storage_type = storage_type;
        if (mode == 2 && hole_every > 0 && b % hole_every == hole_every - 1) {
            lb.block.has_alloc_opts = true;  // allocated, never written, no location: BlockReaderHole
            is_hole[static_cast<size_t>(b)] = 1;
            continue;
        }
        Err e = w->w.store().reserve_block(id, blen, storage_type, g_synth_shard_world >= 1 ? static_cast<int>(b % g_synth_shard_world) : -1,
                                           &targets[static_cast<size_t>(b)]);
        if (e) {
            for (int64_t x = 0; x < b; x++)
                if (!is_hole[static_cast<size_t>(x)]) w->w.store().abort_block(fb.block_locs[static_cast<size_t>(x)].block.id, &targets[static_cast<size_t>(x)]);
            return fail(e);
        }
    }
    std::atomic<int64_t> next{0};
    std::mutex emu;
    Err first;
    const int T = std::max(1, std::min<int>(threads, static_cast<int>(std::max<int64_t>(nb, 1))));
    auto work = [&] {
        std::vector<uint8_t> buf(static_cast<size_t>(std::min(block_size, std::max<int64_t>(len, 1))));
        for (;;) {
            const int64_t b = next.fetch_add(1);
            if (b >= nb) break;
            if (is_hole[static_cast<size_t>(b)]) continue;
            LocatedBlock& lb = fb.block_locs[static_cast<size_t>(b)];
            BlockWriteTarget& t = targets[static_cast<size_t>(b)];
            const int64_t blen = lb.block.len;
            if (!node_cpus.empty()) bind_cpus(node_cpus[static_cast<size_t>(b % g_synth_shard_world) % node_cpus.size()]);
            uint8_t* out = t.arena ? t.mem() : buf.data();
            if (mode == 1)
                for (int64_t o = 0; o < blen; o += static_cast<int64_t>(az.size()))
                    memcpy(out + o, az.data(), static_cast<size_t>(std::min<int64_t>(static_cast<int64_t>(az.size()), blen - o)));
            else
                cv_synth_block(static_cast<uint64_t>(inode_id), static_cast<uint64_t>(b), out, static_cast<size_t>(blen));
            lb.crc32 = cv_host_crc(0, out, static_cast<size_t>(blen));
            lb.crc32c = cv_host_crc(1, out, static_cast<size_t>(blen));
            lb.has_crc = true;
            Err e;
            if (!t.arena) {
                const int fd = ::open(t.path.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
                if (fd < 0) e = Err::io(str_printf("open %s: %s", t.path.c_str(), strerror(errno)));
                for (int64_t done = 0; !e && done < blen;) {
                    const ssize_t wr = ::write(fd, out + done, static_cast<size_t>(blen - done));
                    if (wr < 0 && errno == EINTR) continue;
                    if (wr <= 0) e = Err::io(str_printf("write %s: %s", t.path.c_str(), strerror(errno)));
                    else done += wr;
                }
                if (fd >= 0) ::close(fd);
            }
            if (!e) e = w->w.store().commit_block(lb.block.id, &t, blen);
            lb.block.storage_type = t.dir_storage_type;
            lb.locs.push_back(addr);
            if (e) {
                std::lock_guard<std::mutex> lk(emu);
                if (!first) first = e;
                break;
            }
        }
    };
    std::vector<std::thread> ts;
    for (int t = 0; t < T; t++) ts.emplace_back(work);
    for (auto& t : ts) t.join();
    if (first) return fail(first);
    Namespace ns;
    ns.put(fb);
    const std::string text = ns.dump();
    if (manifest_out) {
        *manifest_out = static_cast<char*>(malloc(text.size() + 1));
        memcpy(*manifest_out, text.c_str(), text.size() + 1);
    }
    return ok();
    API_GUARD_END
}

}  // extern "C"
