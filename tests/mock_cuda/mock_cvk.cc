// TEST INFRASTRUCTURE ONLY -- plain-loop CPU stand-ins for the cvk_* launchers (include/curvine_b200_kernels.h), linked
// into the mock library instead of csrc/kernels.cu so the host pipeline above them can run without a GPU.  They restate
// the launchers' CONTRACT (what lands where, which flags are raised), not the kernels' algorithm: a bytewise table CRC, memcpy.
// The real kernels are checked against the oracle on an H100 by tests/test_kernels_gpu.py; nothing here is ever timed or shipped.
#include <string.h>

#include <atomic>

#include "../../include/curvine_b200_kernels.h"
#include "../../curvine_b200/csrc/crc_gf.h"

namespace {
std::atomic<uint64_t> g_launches{0};
struct Tables {
    uint32_t t[2][256];
    Tables() {
        for (int pid = 0; pid < 2; pid++)
            for (uint32_t v = 0; v < 256; v++) {
                uint32_t r = v;
                for (int k = 0; k < 8; k++) r = cv::gf_mulx(r, cv::poly_of(pid));
                t[pid][v] = r;
            }
    }
};
const Tables& tables() {
    static Tables T;
    return T;
}
uint32_t crc_update(int poly, uint32_t state, const uint8_t* p, uint64_t n) {  // state = running register (pre-inverted)
    const uint32_t* t = tables().t[poly];
    for (uint64_t i = 0; i < n; i++) state = t[(state ^ p[i]) & 0xffu] ^ (state >> 8);
    return state;
}
uint32_t be32(const uint8_t* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }
void put32(uint8_t* p, uint32_t v) { p[0] = v >> 24, p[1] = v >> 16, p[2] = v >> 8, p[3] = v; }
}  // namespace

extern "C" {

int cvk_init(int device) { return device >= 0 && device < 8 ? 0 : 101; }
uint64_t cvk_launch_count(void) { return g_launches.load(); }
int cvk_tune(int, int) { return 0; }
static std::atomic<bool> g_prof_on{false};
static std::atomic<uint32_t> g_prof_n{0};
int cvk_profile_enable(int on) {
    g_prof_on.store(on != 0);
    g_prof_n.store(0);
    return 0;
}
int cvk_profile_collect(double* ms, uint32_t* n) {  // pretend every walker launch took 1 ms: the callers only need non-zero
    const uint32_t k = g_prof_n.exchange(0);
    if (ms) *ms = 1.0 * k;
    if (n) *n = k;
    return 0;
}

int cvk_crc_blocks(const uint8_t* d_base, const uint64_t* d_off, const uint64_t* d_len, uint32_t n, int poly, uint64_t, uint32_t* d_crc_out,
                   cv_stream_t) {
    if (poly != 0 && poly != 1) return 1;
    for (uint32_t i = 0; i < n; i++) d_crc_out[i] = ~crc_update(poly, 0xffffffffu, d_base + d_off[i], d_len[i]);
    g_launches += 5;
    if (g_prof_on.load()) g_prof_n++;
    return 0;
}

int cvk_verify_crcs(const uint32_t* d_crc, const uint32_t* d_expect, uint32_t n, uint32_t* d_n_bad, uint8_t* d_bad_mask, cv_stream_t) {
    for (uint32_t i = 0; i < n; i++) {
        const bool bad = d_crc[i] != d_expect[i];
        if (d_bad_mask) d_bad_mask[i] = bad;
        if (bad) (*d_n_bad)++;
    }
    g_launches++;
    return 0;
}

int cvk_verify_crcs_masked(const uint32_t* d_crc, const uint32_t* d_expect, const uint8_t* d_skip, uint32_t n, uint32_t* d_n_bad, uint8_t* d_bad_mask,
                           cv_stream_t) {
    for (uint32_t i = 0; i < n; i++) {
        const bool bad = !(d_skip && d_skip[i]) && d_crc[i] != d_expect[i];
        if (d_bad_mask) d_bad_mask[i] = bad;
        if (bad) (*d_n_bad)++;
    }
    g_launches++;
    return 0;
}

int cvk_expand_streams(const CvStreamDesc* s, uint32_t n_streams, CvFrameDesc* out, uint32_t n_frames, cv_stream_t) {
    for (uint32_t i = 0; i < n_streams; i++) {
        const CvStreamDesc& d = s[i];
        const uint64_t nf = d.block_len ? (d.block_len + d.chunk_size - 1) / d.chunk_size : 0;
        for (uint64_t f = 0; f < nf; f++) {
            const uint64_t idx = uint64_t(d.first_frame) + f;
            if (idx >= n_frames) break;
            CvFrameDesc o;
            memset(&o, 0, sizeof(o));
            o.wire_off = d.wire_off + f * (uint64_t(CV_PROTOCOL_SIZE) + d.chunk_size);
            o.dst_off = d.dst_off + f * d.chunk_size;
            const uint64_t rem = d.block_len - f * d.chunk_size;
            o.data_len = static_cast<uint32_t>(rem < d.chunk_size ? rem : d.chunk_size);
            o.req_id = d.req_id, o.seq_id = d.first_seq_id + static_cast<int32_t>(f), o.block = d.block, o.code = d.code, o.status = d.status;
            o.tail_clip = f + 1 == nf ? d.tail_clip : 0;
            out[idx] = o;
        }
    }
    g_launches++;
    return 0;
}

int cvk_unpack_frames(const uint8_t* d_wire, const CvFrameDesc* d_desc, uint32_t n_frames, uint32_t n_blocks, uint8_t* d_dst, int poly, uint64_t,
                      uint32_t* d_block_crc, uint32_t* d_err_flags, cv_stream_t) {
    if (poly != 0 && poly != 1) return 1;
    uint32_t state = 0xffffffffu, cur = 0xffffffffu;
    for (uint32_t b = 0; d_block_crc && b < n_blocks; b++) d_block_crc[b] = 0;  // CRC of zero bytes
    for (uint32_t i = 0; i < n_frames; i++) {
        const CvFrameDesc& d = d_desc[i];
        const uint8_t* f = d_wire + d.wire_off;
        const int32_t total_len = static_cast<int32_t>(be32(f)), header_len = static_cast<int32_t>(be32(f + 4));
        const int64_t req_id = static_cast<int64_t>((uint64_t(be32(f + 10)) << 32) | be32(f + 14));
        const int32_t seq_id = static_cast<int32_t>(be32(f + 18));
        const int64_t data_len = int64_t(total_len) - header_len - CV_HEAD_SIZE;
        uint32_t e = 0;
        if (data_len < 0 || data_len > CV_MAX_DATA_SIZE) e |= CV_FERR_DATA_RANGE;
        if (int64_t(total_len) != int64_t(CV_HEAD_SIZE) + d.header_len + d.data_len) e |= CV_FERR_TOTAL_LEN;
        if (header_len != static_cast<int32_t>(d.header_len)) e |= CV_FERR_HEADER_LEN;
        if (f[8] != d.code) e |= CV_FERR_CODE;
        if (f[9] != d.status) e |= CV_FERR_STATUS;
        if (req_id != d.req_id) e |= CV_FERR_REQ_ID;
        if (seq_id != d.seq_id) e |= CV_FERR_SEQ_ID;
        if (d_err_flags) d_err_flags[i] = e;
        const uint8_t* payload = f + CV_PROTOCOL_SIZE + d.header_len;
        const uint32_t take = d.data_len - (d.tail_clip < d.data_len ? d.tail_clip : d.data_len);
        memmove(d_dst + d.dst_off, payload, take);
        if (d_block_crc && d.block < n_blocks) {
            if (d.block != cur) state = 0xffffffffu, cur = d.block;
            state = crc_update(poly, state, payload, take);
            d_block_crc[d.block] = ~state;
        }
    }
    g_launches += 6;
    return 0;
}

int cvk_pack_frames(const uint8_t* d_src, const CvFrameDesc* d_desc, uint32_t n_frames, uint32_t n_blocks, uint8_t* d_wire, int poly, uint64_t,
                    uint32_t* d_block_crc, cv_stream_t) {
    if (poly != 0 && poly != 1) return 1;
    uint32_t state = 0xffffffffu, cur = 0xffffffffu;
    for (uint32_t b = 0; d_block_crc && b < n_blocks; b++) d_block_crc[b] = 0;
    for (uint32_t i = 0; i < n_frames; i++) {
        const CvFrameDesc& d = d_desc[i];
        uint8_t* f = d_wire + d.wire_off;
        put32(f, CV_HEAD_SIZE + d.data_len), put32(f + 4, 0);
        f[8] = d.code, f[9] = d.status;
        put32(f + 10, static_cast<uint32_t>(static_cast<uint64_t>(d.req_id) >> 32)), put32(f + 14, static_cast<uint32_t>(d.req_id));
        put32(f + 18, static_cast<uint32_t>(d.seq_id));
        memmove(f + CV_PROTOCOL_SIZE, d_src + d.dst_off, d.data_len);
        if (d_block_crc && d.block < n_blocks) {
            if (d.block != cur) state = 0xffffffffu, cur = d.block;
            state = crc_update(poly, state, d_src + d.dst_off, d.data_len);
            d_block_crc[d.block] = ~state;
        }
    }
    g_launches += 6;
    return 0;
}

int cvk_gather_pages(const uint8_t* d_src, const CvSeg* d_segs, uint32_t n, uint64_t, uint8_t* d_dst, cv_stream_t) {
    for (uint32_t i = 0; i < n; i++) memmove(d_dst + d_segs[i].dst_off, d_src + d_segs[i].src_off, d_segs[i].len);
    g_launches += 4;
    return 0;
}

int cvk_deinterleave_blocks(const uint8_t* g, uint64_t shard_stride, uint32_t world, uint64_t block_size, uint64_t n_blocks, uint64_t file_len,
                            uint8_t* d_dst, cv_stream_t) {
    if (world == 0 || block_size == 0) return 1;
    for (uint64_t b = 0; b < n_blocks; b++) {
        const uint64_t start = b * block_size;
        if (start >= file_len) break;
        const uint64_t len = file_len - start < block_size ? file_len - start : block_size;
        memmove(d_dst + start, g + (b % world) * shard_stride + (b / world) * block_size, len);
    }
    g_launches += 4;
    return 0;
}

int cvk_gather_shards_p2p(const uint8_t* const* shard_ptrs, uint32_t world, uint64_t block_size, uint64_t n_blocks, uint64_t file_len, uint8_t* d_dst,
                          cv_stream_t) {
    if (world == 0 || block_size == 0) return 1;
    for (uint64_t b = 0; b < n_blocks; b++) {
        const uint64_t start = b * block_size;
        if (start >= file_len) break;
        const uint64_t len = file_len - start < block_size ? file_len - start : block_size;
        memmove(d_dst + start, shard_ptrs[b % world] + (b / world) * block_size, len);
    }
    g_launches += 4;
    return 0;
}
}
