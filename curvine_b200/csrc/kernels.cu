// sm_90a kernels for the Curvine sequential block-read path + their extern "C" launchers
// (declared in include/curvine_b200_kernels.h, which cites the reference code each one replaces).
//
// This is a byte-stream / integer path: no tensor cores.  Design (see DESIGN.md §3):
//   * CRC is linear over GF(2).  Each warp owns a contiguous *segment* and walks it in 512-byte rows
//     (one coalesced 16-byte vector per lane).  Every lane keeps 4 independent 32-bit Horner chains
//     (one per word of its vector): a <- a * x^4096 (+) w.  The multiply by the row constant x^4096 is
//     4 shared-memory lookups; the tables are replicated per lane ([table][byte][lane]) so bank == lane and
//     the data-dependent lookups are bank-conflict free.
//   * A segment ends with one fold per lane (weights x^(128*e)) and a warp-shuffle XOR reduction.
//   * Segment partials are folded per block (Horner with x^(8*SEG)) by a tiny second kernel, which also
//     applies init/xorout, so results are bit-identical to crc32fast / zlib (or CRC-32C).
//   * The same row walker optionally stores the (re-aligned) vectors to a destination, which gives the
//     fused frame-unpack+gather+CRC (K2), frame-pack+CRC (K4) and page scatter/gather (K3) kernels.
// Launch train of one call: prep_* (piece geometry) -> scan_counts (prefix sum of per-piece unit counts) -> expand_units
// (one 32-byte record per unit) -> walk_kernel (persistent: one 1024-thread CTA per SM, 132 on H100 SXM, contiguous unit range per
// CTA, a warp per unit) -> fold_blocks (unit partials -> one CRC per block).  Workspaces come from a private memory pool.
#include <cuda_runtime.h>

#include <atomic>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/curvine_b200_kernels.h"
#include "crc_gf.h"

namespace cv {

struct Piece {
    const uint8_t* src;
    uint8_t* dst;  // nullptr when there is nothing to store
    uint64_t len;
};

struct Geom {
    uint32_t head;   // bytes before the first 16-byte aligned anchor address
    uint32_t tail;   // bytes after the last whole 16-byte vector
    uint64_t body;   // multiple of 16
    uint32_t nseg;   // ceil(body / SEG)
    uint32_t units;  // max(1, nseg) if len > 0 else 0
};

template <bool DST>
__device__ __forceinline__ Geom piece_geom(const Piece& p, uint32_t seg_shift) {
    Geom g;
    const uintptr_t anchor = DST ? reinterpret_cast<uintptr_t>(p.dst) : reinterpret_cast<uintptr_t>(p.src);
    uint32_t head = (16u - static_cast<uint32_t>(anchor & 15u)) & 15u;
    if (head > p.len) head = static_cast<uint32_t>(p.len);
    const uint64_t rest = p.len - head;
    g.head = head;
    g.body = rest & ~15ull;
    g.tail = static_cast<uint32_t>(rest - g.body);
    g.nseg = static_cast<uint32_t>((g.body + ((1ull << seg_shift) - 1)) >> seg_shift);
    g.units = p.len ? (g.nseg ? g.nseg : 1u) : 0u;
    return g;
}

// One unit of walker work, expanded from (pieces, prefix) by expand_units_kernel so that the walker reads ONE 32-byte
// record per unit -- at an address it knows a whole unit ahead, so the record is prefetched behind the current walk
// instead of a chain of dependent lookups (prefix search -> piece -> geometry) stalling the warp at every unit boundary.
struct __align__(16) Unit {
    const uint8_t* src;  // first body byte of the segment (piece.src + head + segment offset)
    uint8_t* dst;        // 16-byte aligned when the walk stores; nullptr otherwise
    uint32_t L;          // body bytes in this segment (multiple of 16; 0 for a piece shorter than one vector)
    uint32_t piece;
    uint32_t head;       // > 0 on the first unit of a piece with head bytes (they sit right before src)
    uint32_t tail;       // > 0 on the last unit of a piece with tail bytes (they sit right behind src + L)
};
static_assert(sizeof(Unit) == 32, "Unit is two 16-byte vectors");

// ------------------------------------------------------------------ piece preparation kernels

__global__ void prep_blocks_kernel(const uint8_t* base, const uint64_t* off, const uint64_t* len, uint32_t n,
                                   uint32_t seg_shift, Piece* pieces, uint32_t* counts) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Piece p{base + off[i], nullptr, len[i]};
    pieces[i] = p;
    counts[i] = piece_geom<false>(p, seg_shift).units;
}

__device__ __forceinline__ uint32_t be32(const uint8_t* p) {
    return (uint32_t(__ldg(p)) << 24) | (uint32_t(__ldg(p + 1)) << 16) | (uint32_t(__ldg(p + 2)) << 8) |
           uint32_t(__ldg(p + 3));
}

// K2 front end: RpcMessage::decode_protocol + RawClient::check_response for every frame in parallel.
__global__ void prep_unpack_kernel(const uint8_t* wire, const CvFrameDesc* desc, uint32_t n, uint8_t* dst,
                                   uint32_t seg_shift, Piece* pieces, uint32_t* counts, uint32_t* err_flags) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const CvFrameDesc d = desc[i];
    const uint8_t* f = wire + d.wire_off;
    const int32_t total_len = static_cast<int32_t>(be32(f));
    const int32_t header_len = static_cast<int32_t>(be32(f + 4));
    const uint8_t code = __ldg(f + 8), status = __ldg(f + 9);
    const int64_t req_id = static_cast<int64_t>((uint64_t(be32(f + 10)) << 32) | be32(f + 14));
    const int32_t seq_id = static_cast<int32_t>(be32(f + 18));
    const int64_t data_len = int64_t(total_len) - header_len - CV_HEAD_SIZE;
    uint32_t e = 0;
    if (data_len < 0 || data_len > CV_MAX_DATA_SIZE) e |= CV_FERR_DATA_RANGE;
    if (int64_t(total_len) != int64_t(CV_HEAD_SIZE) + d.header_len + d.data_len) e |= CV_FERR_TOTAL_LEN;
    if (header_len != static_cast<int32_t>(d.header_len)) e |= CV_FERR_HEADER_LEN;
    if (code != d.code) e |= CV_FERR_CODE;
    if (status != d.status) e |= CV_FERR_STATUS;
    if (req_id != d.req_id) e |= CV_FERR_REQ_ID;
    if (seq_id != d.seq_id) e |= CV_FERR_SEQ_ID;
    if (err_flags) err_flags[i] = e;
    Piece p{f + CV_PROTOCOL_SIZE + d.header_len, dst + d.dst_off, d.data_len - (d.tail_clip < d.data_len ? d.tail_clip : d.data_len)};
    pieces[i] = p;
    counts[i] = piece_geom<true>(p, seg_shift).units;
}

// K4 front end: RpcMessage::encode_protocol for every frame in parallel (big-endian prefix, no header).
__global__ void prep_pack_kernel(const uint8_t* src, const CvFrameDesc* desc, uint32_t n, uint8_t* wire,
                                 uint32_t seg_shift, Piece* pieces, uint32_t* counts) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const CvFrameDesc d = desc[i];
    uint8_t* f = wire + d.wire_off;
    const uint32_t total_len = CV_HEAD_SIZE + d.data_len;
    const uint64_t rid = static_cast<uint64_t>(d.req_id);
    const uint32_t sid = static_cast<uint32_t>(d.seq_id);
    f[0] = total_len >> 24, f[1] = total_len >> 16, f[2] = total_len >> 8, f[3] = total_len;
    f[4] = f[5] = f[6] = f[7] = 0;
    f[8] = d.code, f[9] = d.status;
#pragma unroll
    for (int k = 0; k < 8; k++) f[10 + k] = static_cast<uint8_t>(rid >> (56 - 8 * k));
    f[18] = sid >> 24, f[19] = sid >> 16, f[20] = sid >> 8, f[21] = sid;
    Piece p{src + d.dst_off, f + CV_PROTOCOL_SIZE, d.data_len};
    pieces[i] = p;
    counts[i] = piece_geom<true>(p, seg_shift).units;
}

__global__ void prep_segs_kernel(const uint8_t* src, const CvSeg* segs, uint32_t n, uint8_t* dst, uint32_t seg_shift,
                                 Piece* pieces, uint32_t* counts) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const CvSeg s = segs[i];
    Piece p{src + s.src_off, dst + s.dst_off, s.len};
    pieces[i] = p;
    counts[i] = piece_geom<true>(p, seg_shift).units;
}

// K3 over 2D descriptors, one train: rows [base, base + cnt) of the row numbering row_pref gives (descriptor d owns rows
// [row_pref[d], row_pref[d + 1])).  One warp per descriptor, lanes stride over its rows inside the train, one piece per row.
__global__ void prep_strided_kernel(const uint8_t* src, const CvStridedSeg* segs, const uint64_t* row_pref, uint32_t n, uint8_t* dst,
                                    uint64_t base, uint32_t cnt, uint32_t seg_shift, Piece* pieces, uint32_t* counts) {
    const uint32_t d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (d >= n) return;
    const uint64_t r0 = row_pref[d], r1 = row_pref[d + 1];
    const uint64_t lo = r0 > base ? r0 : base, hi = r1 < base + cnt ? r1 : base + cnt;
    if (lo >= hi) return;
    const CvStridedSeg s = segs[d];
    for (uint64_t g = lo + lane; g < hi; g += 32) {
        const uint64_t k = g - r0;
        Piece p{src + s.src_off + k * s.src_pitch, dst + s.dst_off + k * s.dst_pitch, s.len};
        pieces[g - base] = p;
        counts[g - base] = piece_geom<true>(p, seg_shift).units;
    }
}

__global__ void prep_deinterleave_kernel(const uint8_t* gathered, uint64_t shard_stride, uint32_t world,
                                         uint64_t block_size, uint64_t n_blocks, uint64_t file_len, uint8_t* dst,
                                         uint32_t seg_shift, Piece* pieces, uint32_t* counts) {
    const uint64_t b = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (b >= n_blocks) return;
    const uint64_t start = b * block_size;
    const uint64_t len = start >= file_len ? 0 : (file_len - start < block_size ? file_len - start : block_size);
    Piece p{gathered + (b % world) * shard_stride + (b / world) * block_size, dst + start, len};
    pieces[b] = p;
    counts[b] = piece_geom<true>(p, seg_shift).units;
}

// Like prep_deinterleave_kernel, but every rank's shard has its own base pointer (peer memory mapped over NVLink).
__global__ void prep_gather_shards_kernel(const uint8_t* const* shard_ptrs, uint32_t world, uint64_t block_size, uint64_t n_blocks,
                                          uint64_t file_len, uint8_t* dst, uint32_t seg_shift, Piece* pieces, uint32_t* counts) {
    const uint64_t b = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (b >= n_blocks) return;
    const uint64_t start = b * block_size;
    const uint64_t len = start >= file_len ? 0 : (file_len - start < block_size ? file_len - start : block_size);
    Piece p{shard_ptrs[b % world] + (b / world) * block_size, dst + start, len};
    pieces[b] = p;
    counts[b] = piece_geom<true>(p, seg_shift).units;
}

__global__ void expand_streams_kernel(const CvStreamDesc* streams, uint32_t n_streams, CvFrameDesc* out,
                                      uint32_t n_frames) {
    // one warp per stream, lanes stride over its frames
    const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (s >= n_streams) return;
    const CvStreamDesc d = streams[s];
    const uint64_t nf = d.block_len ? (d.block_len + d.chunk_size - 1) / d.chunk_size : 0;
    for (uint64_t f = lane; f < nf; f += 32) {
        const uint64_t idx = uint64_t(d.first_frame) + f;
        if (idx >= n_frames) break;
        CvFrameDesc o;
        o.wire_off = d.wire_off + f * (uint64_t(CV_PROTOCOL_SIZE) + d.chunk_size);
        o.dst_off = d.dst_off + f * d.chunk_size;
        const uint64_t rem = d.block_len - f * d.chunk_size;
        o.data_len = static_cast<uint32_t>(rem < d.chunk_size ? rem : d.chunk_size);
        o.header_len = 0;
        o.req_id = d.req_id;
        o.seq_id = d.first_seq_id + static_cast<int32_t>(f);
        o.block = d.block;
        o.code = d.code;
        o.status = d.status;
        o.pad_[0] = o.pad_[1] = 0;
        o.tail_clip = f + 1 == nf ? d.tail_clip : 0;
        out[idx] = o;
    }
}

// first[b] / last[b]: frame range of block b (frames of a block are contiguous); zero-initialised by the caller
__global__ void mark_block_ranges_kernel(const CvFrameDesc* desc, uint32_t n, uint32_t n_blocks, uint32_t* first,
                                         uint32_t* last) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t b = desc[i].block;
    if (b >= n_blocks) return;
    if (i == 0 || desc[i - 1].block != b) first[b] = i;
    if (i == n - 1 || desc[i + 1].block != b) last[b] = i + 1;
}

// exclusive prefix sum of counts[0..n) into prefix[0..n]; single CTA (n is a frame/block/page count, not bytes).
// Tiles of 4096 elements: every thread takes one 16-byte vector of four counts (coalesced), the tile is scanned with
// warp shuffles + one shared-memory hop, and the next tile's vector is already in flight while the current one is
// scanned.  256 Ki page descriptors (a 1 GiB FUSE-shaped gather) scan in ~64 tile steps.
__global__ void __launch_bounds__(1024) scan_counts_kernel(const uint32_t* __restrict__ counts, uint32_t n, uint32_t* __restrict__ prefix) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t tile_total;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    auto load4 = [&](uint32_t base) -> uint4 {  // counts[base .. base+3], zero past n (counts is 256-byte aligned)
        if (base + 4 <= n) return __ldg(reinterpret_cast<const uint4*>(counts + base));
        uint4 v = make_uint4(0, 0, 0, 0);
        if (base < n) v.x = __ldg(counts + base);
        if (base + 1 < n) v.y = __ldg(counts + base + 1);
        if (base + 2 < n) v.z = __ldg(counts + base + 2);
        return v;
    };
    uint32_t carry = 0;
    uint4 nxt = load4(tid * 4);
    for (uint32_t t0 = 0; t0 < n; t0 += 4096) {
        const uint4 c = nxt;
        const uint32_t base = t0 + tid * 4;
        if (t0 + 4096 < n) nxt = load4(base + 4096);
        const uint32_t sum = c.x + c.y + c.z + c.w;
        uint32_t incl = sum;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const uint32_t w = warp_sums[lane];
            uint32_t wi = w;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, wi, d);
                if (lane >= d) wi += t;
            }
            warp_sums[lane] = wi - w;  // exclusive
            if (lane == 31) tile_total = wi;
        }
        __syncthreads();
        const uint32_t e0 = carry + warp_sums[warp] + incl - sum;  // exclusive prefix of this thread's first element
        const uint4 o = make_uint4(e0, e0 + c.x, e0 + c.x + c.y, e0 + c.x + c.y + c.z);
        if (base + 4 <= n) {
            *reinterpret_cast<uint4*>(prefix + base) = o;
        } else {
            if (base < n) prefix[base] = o.x;
            if (base + 1 < n) prefix[base + 1] = o.y;
            if (base + 2 < n) prefix[base + 2] = o.z;
        }
        carry += tile_total;
        __syncthreads();  // warp_sums / tile_total are rewritten by the next tile
    }
    if (tid == 0) prefix[n] = carry;
}

// Many pieces (a FUSE-shaped gather has one per 4 KiB page: 262,144 for 1 GiB): the single-CTA scan above takes longer than the
// copy it prepares.  Two parallel launches instead: every CTA sums its tile of 4096 counts; then every CTA adds up the tile sums
// before its own (at most a few hundred values) and scans its tile from that carry.
__device__ __forceinline__ uint32_t block_sum_1024(uint32_t v, uint32_t* sh) {  // sh: 32 words; result valid in every thread
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    uint32_t t = sh[lane];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) t += __shfl_xor_sync(0xffffffffu, t, d);
    __syncthreads();
    return t;
}

__global__ void __launch_bounds__(1024) tile_sums_kernel(const uint32_t* __restrict__ counts, uint32_t n, uint32_t* __restrict__ sums) {
    __shared__ uint32_t sh[32];
    const uint32_t base = blockIdx.x * 4096u + threadIdx.x * 4;
    uint32_t v = 0;
    if (base + 4 <= n) {
        const uint4 c = __ldg(reinterpret_cast<const uint4*>(counts + base));
        v = c.x + c.y + c.z + c.w;
    } else {
        for (uint32_t k = 0; k < 4; k++)
            if (base + k < n) v += __ldg(counts + base + k);
    }
    const uint32_t t = block_sum_1024(v, sh);
    if (threadIdx.x == 0) sums[blockIdx.x] = t;
}

__global__ void __launch_bounds__(1024) scan_tiles_kernel(const uint32_t* __restrict__ counts, uint32_t n, const uint32_t* __restrict__ sums,
                                                          uint32_t* __restrict__ prefix) {
    __shared__ uint32_t sh[32];
    __shared__ uint32_t warp_sums[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t before = 0;
    for (uint32_t i = tid; i < blockIdx.x; i += 1024) before += __ldg(sums + i);
    const uint32_t carry = block_sum_1024(before, sh);
    const uint32_t base = blockIdx.x * 4096u + tid * 4;
    uint4 c = make_uint4(0, 0, 0, 0);
    if (base + 4 <= n) c = __ldg(reinterpret_cast<const uint4*>(counts + base));
    else {
        if (base < n) c.x = __ldg(counts + base);
        if (base + 1 < n) c.y = __ldg(counts + base + 1);
        if (base + 2 < n) c.z = __ldg(counts + base + 2);
    }
    const uint32_t sum = c.x + c.y + c.z + c.w;
    uint32_t incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const uint32_t w = warp_sums[lane];
        uint32_t wi = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, wi, d);
            if (lane >= d) wi += t;
        }
        warp_sums[lane] = wi - w;  // exclusive
    }
    __syncthreads();
    const uint32_t e0 = carry + warp_sums[warp] + incl - sum;
    const uint4 o = make_uint4(e0, e0 + c.x, e0 + c.x + c.y, e0 + c.x + c.y + c.z);
    if (base + 4 <= n) {
        *reinterpret_cast<uint4*>(prefix + base) = o;
    } else {
        if (base < n) prefix[base] = o.x;
        if (base + 1 < n) prefix[base + 1] = o.y;
        if (base + 2 < n) prefix[base + 2] = o.z;
    }
    // the thread that holds element n-1 also writes the total
    if (base < n && base + 4 >= n) prefix[n] = e0 + sum;
}

// ------------------------------------------------------------------ the row walker

constexpr uint32_t kTmWords = 4 * 256 * 32;  // replicated x^4096 tables: [table][byte][lane]
constexpr uint32_t kSmemWords = kTmWords + 256 + 64 + 16;
constexpr uint32_t kSmemBytes = kSmemWords * 4;

__device__ __forceinline__ uint4 ld_stream(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// a * x^4096 mod P: four conflict-free shared-memory lookups.  tb = shared byte address of the lane's
// column (tables + lane*4); entry (table t, byte v) lives at tb + t*32768 + v*128.  Byte extraction is a PRMT
// (ALU pipe) and the scale-and-add an IMAD (FMA pipe) so the two integer pipes share the address math.
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t mul_row(uint32_t a, uint32_t tb) {
    const uint32_t i0 = __byte_perm(a, 0, 0x4440) * 128u + tb;
    const uint32_t i1 = __byte_perm(a, 0, 0x4441) * 128u + tb;
    const uint32_t i2 = __byte_perm(a, 0, 0x4442) * 128u + tb;
    const uint32_t i3 = __byte_perm(a, 0, 0x4443) * 128u + tb;
    return lds_u32(i0) ^ lds_u32(i1 + 32768u) ^ lds_u32(i2 + 65536u) ^ lds_u32(i3 + 98304u);
}

// y * x^32 mod P via the byte table
__device__ __forceinline__ uint32_t mul_word(uint32_t y, const uint32_t* t0) {
#pragma unroll
    for (int k = 0; k < 4; k++) y = t0[y & 0xffu] ^ (y >> 8);
    return y;
}

// raw CRC (init 0, no xorout) of one 16-byte vector
__device__ __forceinline__ uint32_t raw_vec(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, const uint32_t* t0) {
    uint32_t r = mul_word(w0, t0);
    r = mul_word(r ^ w1, t0);
    r = mul_word(r ^ w2, t0);
    return mul_word(r ^ w3, t0);
}

// plain (coherent-path) 16-byte load: the source of a DST walk may be PEER memory mapped over NVLink
// (cvk_gather_shards_p2p), where the non-coherent ld.global.nc path faults
__device__ __forceinline__ uint4 ld_plain(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// 16-byte store to GLOBAL memory.  The walkers' destination pointer lives in the unit table as a generic pointer, so a plain
// `*p = v` compiles to a generic ST.E.128 (address-space check per store); every destination here is global memory.
__device__ __forceinline__ void st_vec(uint4* p, const uint4& v) {
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// One output vector of a shifted walk: 16 bytes starting Q words + r8 bits into the 8-word window [ra | nb].
template <int Q>
__device__ __forceinline__ uint4 shift_window(const uint4& ra, const uint4& nb, uint32_t r8) {
    uint4 v;
    if (Q == 0) {
        v.x = __funnelshift_r(ra.x, ra.y, r8), v.y = __funnelshift_r(ra.y, ra.z, r8);
        v.z = __funnelshift_r(ra.z, ra.w, r8), v.w = __funnelshift_r(ra.w, nb.x, r8);
    } else if (Q == 1) {
        v.x = __funnelshift_r(ra.y, ra.z, r8), v.y = __funnelshift_r(ra.z, ra.w, r8);
        v.z = __funnelshift_r(ra.w, nb.x, r8), v.w = __funnelshift_r(nb.x, nb.y, r8);
    } else if (Q == 2) {
        v.x = __funnelshift_r(ra.z, ra.w, r8), v.y = __funnelshift_r(ra.w, nb.x, r8);
        v.z = __funnelshift_r(nb.x, nb.y, r8), v.w = __funnelshift_r(nb.y, nb.z, r8);
    } else {
        v.x = __funnelshift_r(ra.w, nb.x, r8), v.y = __funnelshift_r(nb.x, nb.y, r8);
        v.z = __funnelshift_r(nb.y, nb.z, r8), v.w = __funnelshift_r(nb.z, nb.w, r8);
    }
    return v;
}

// The right neighbour's aligned vector (lane 31 takes `wrap`, the first vector of the following row, from lane 0).
// Only the words the window for Q reaches are exchanged.
template <int Q>
__device__ __forceinline__ uint4 take_right(const uint4& own, const uint4& wrap, uint32_t lane) {
    const uint32_t from = (lane + 1) & 31;
    uint4 nb = make_uint4(0, 0, 0, 0);
    nb.x = __shfl_sync(0xffffffffu, lane == 0 ? wrap.x : own.x, from);
    if (Q >= 1) nb.y = __shfl_sync(0xffffffffu, lane == 0 ? wrap.y : own.y, from);
    if (Q >= 2) nb.z = __shfl_sync(0xffffffffu, lane == 0 ? wrap.z : own.z, from);
    if (Q >= 3) nb.w = __shfl_sync(0xffffffffu, lane == 0 ? wrap.w : own.w, from);
    return nb;
}

#define CV_STEP(v)                       \
    do {                                 \
        a0 = mul_row(a0, tl) ^ (v).x;    \
        a1 = mul_row(a1, tl) ^ (v).y;    \
        a2 = mul_row(a2, tl) ^ (v).z;    \
        a3 = mul_row(a3, tl) ^ (v).w;    \
    } while (0)

struct Chains {
    uint32_t a0, a1, a2, a3;
    uint4 vr;  // the partial last row's vector (zero when the lane has none)
};

// Shifted source (every frame payload: 22-byte prefixes put it 6, 12, 2, 8, ... bytes off the destination's phase).
// Each ALIGNED source vector is loaded exactly once; the 16 output bytes of a lane straddle its own vector and its
// right neighbour's, which arrives by warp shuffle.  Rows go in tiles of T: T row loads plus one single-lane load (the
// vector that follows the tile, needed by lane 31 of its last row) are issued back to back, so a warp keeps T*512 bytes
// in flight; rows of a tile are independent of each other.  Q = word part of the shift (template: the window
// selection and the number of shuffles are resolved at compile time), r8 = its bit part.
template <bool CRC, int T, int Q>
__device__ __forceinline__ void walk_shifted(const uint8_t* src, uint8_t* dst, uint32_t L, uint32_t lane, uint32_t tl, Chains& c) {
    const uint32_t sh = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(src) & 15u);
    const uint4* bp = reinterpret_cast<const uint4*>(src - sh) + lane;
    uint4* dp = reinterpret_cast<uint4*>(dst) + lane;
    const uint32_t R = L >> 9, nv = (L & 511u) >> 4;
    const uint32_t nvec = (L >> 4) + 1;  // aligned vectors that hold the L bytes
    const uint32_t rows = R + (nv ? 1u : 0u);
    const uint32_t r8 = (sh & 3u) * 8u;
    const uint4 zero = make_uint4(0, 0, 0, 0);
    uint32_t a0 = c.a0, a1 = c.a1, a2 = c.a2, a3 = c.a3;
    uint32_t j = 0;
    for (; j + T <= R; j += T) {  // whole tiles: every vector touched (incl. the one after the tile) is < nvec
        uint4 ra[T];
#pragma unroll
        for (int k = 0; k < T; k++) ra[k] = ld_plain(bp + (j + k) * 32);
        uint4 ex = zero;
        if (lane == 0) ex = ld_plain(bp + (j + T) * 32);
#pragma unroll
        for (int k = 0; k < T; k++) {
            const uint4 nb = take_right<Q>(ra[k], k + 1 < T ? ra[(k + 1) % T] : ex, lane);
            const uint4 v = shift_window<Q>(ra[k], nb, r8);
            st_vec(dp + (j + k) * 32, v);
            if (CRC) CV_STEP(v);
        }
    }
    for (; j < rows; j++) {  // leftover rows, bounds-checked
        const uint4 ra = j * 32 + lane < nvec ? ld_plain(bp + j * 32) : zero;
        uint4 ex = zero;
        if (lane == 0 && (j + 1) * 32 < nvec) ex = ld_plain(bp + (j + 1) * 32);
        const uint4 nb = take_right<Q>(ra, ex, lane);
        const uint4 v = shift_window<Q>(ra, nb, r8);
        if (j < R) {
            st_vec(dp + j * 32, v);
            if (CRC) CV_STEP(v);
        } else if (lane < nv) {
            st_vec(dp + j * 32, v);
            c.vr = v;
        }
    }
    c.a0 = a0, c.a1 = a1, c.a2 = a2, c.a3 = a3;
}

// Source and destination share their 16-byte phase: one load and one store per vector, tiles of T rows.
template <bool CRC, int T>
__device__ __forceinline__ void walk_aligned_copy(const uint8_t* src, uint8_t* dst, uint32_t L, uint32_t lane, uint32_t tl, Chains& c) {
    const uint4* sp = reinterpret_cast<const uint4*>(src) + lane;
    uint4* dp = reinterpret_cast<uint4*>(dst) + lane;
    const uint32_t R = L >> 9, nv = (L & 511u) >> 4;
    uint32_t a0 = c.a0, a1 = c.a1, a2 = c.a2, a3 = c.a3;
    uint32_t j = 0;
    for (; j + T <= R; j += T) {
        uint4 v[T];
#pragma unroll
        for (int k = 0; k < T; k++) v[k] = ld_plain(sp + (j + k) * 32);
#pragma unroll
        for (int k = 0; k < T; k++) {
            st_vec(dp + (j + k) * 32, v[k]);
            if (CRC) CV_STEP(v[k]);
        }
    }
    for (; j < R; j++) {
        const uint4 v = ld_plain(sp + j * 32);
        st_vec(dp + j * 32, v);
        if (CRC) CV_STEP(v);
    }
    if (lane < nv) {
        c.vr = ld_plain(sp + R * 32);
        st_vec(dp + R * 32, c.vr);
    }
    c.a0 = a0, c.a1 = a1, c.a2 = a2, c.a3 = a3;
}

// One warp walks L bytes (multiple of 16) starting at src (dst is 16-byte aligned when DST; src is 16-byte
// aligned when !DST).  Returns the segment's raw CRC in every lane (0 when !CRC).  T = rows per tile of the DST walks.
template <bool CRC, bool DST, int T>
__device__ __forceinline__ uint32_t walk_segment(const uint8_t* src, uint8_t* dst, uint32_t L, uint32_t lane,
                                                 const uint32_t* smem, uint32_t poly) {
    const uint32_t tl = static_cast<uint32_t>(__cvta_generic_to_shared(smem)) + lane * 4u;
    const uint32_t* t0 = smem + kTmWords;
    const uint32_t* xp128 = t0 + 256;
    const uint32_t nv = (L & 511u) >> 4;
    Chains c;
    c.a0 = c.a1 = c.a2 = c.a3 = 0;
    c.vr = make_uint4(0, 0, 0, 0);

    if (!DST) {
        const uint32_t R = L >> 9;
        uint32_t a0 = 0, a1 = 0, a2 = 0, a3 = 0;
        const uint4* sp = reinterpret_cast<const uint4*>(src) + lane;
        uint32_t j = 0;
        for (; j + 4 <= R; j += 4) {
            const uint4 v0 = ld_stream(sp + (j + 0) * 32);
            const uint4 v1 = ld_stream(sp + (j + 1) * 32);
            const uint4 v2 = ld_stream(sp + (j + 2) * 32);
            const uint4 v3 = ld_stream(sp + (j + 3) * 32);
            CV_STEP(v0);
            CV_STEP(v1);
            CV_STEP(v2);
            CV_STEP(v3);
        }
        for (; j < R; j++) {
            const uint4 v = ld_stream(sp + j * 32);
            CV_STEP(v);
        }
        if (lane < nv) c.vr = ld_stream(sp + R * 32);
        c.a0 = a0, c.a1 = a1, c.a2 = a2, c.a3 = a3;
    } else {
        const uint32_t sh = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(src) & 15u);
        if (sh == 0) {
            walk_aligned_copy<CRC, T>(src, dst, L, lane, tl, c);
        } else {
            switch (sh >> 2) {  // warp-uniform
                case 0: walk_shifted<CRC, T, 0>(src, dst, L, lane, tl, c); break;
                case 1: walk_shifted<CRC, T, 1>(src, dst, L, lane, tl, c); break;
                case 2: walk_shifted<CRC, T, 2>(src, dst, L, lane, tl, c); break;
                default: walk_shifted<CRC, T, 3>(src, dst, L, lane, tl, c); break;
            }
        }
    }
    if (!CRC) return 0;
    // lane fold: rows weigh x^(128*(31-lane+nv)), the partial row x^(128*(nv-1-lane))
    uint32_t t = gf_mul(raw_vec(c.a0, c.a1, c.a2, c.a3, t0), xp128[31u - lane + nv], poly);
    if (lane < nv) t ^= gf_mul(raw_vec(c.vr.x, c.vr.y, c.vr.z, c.vr.w, t0), xp128[nv - 1u - lane], poly);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) t ^= __shfl_xor_sync(0xffffffffu, t, d);
    return t;
}

// bytewise raw CRC (+ optional copy) of a short run; single lane
template <bool CRC, bool DST>
__device__ __forceinline__ uint32_t walk_bytes(const uint8_t* src, uint8_t* dst, uint32_t n, const uint32_t* t0) {
    uint32_t r = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t b = DST ? *reinterpret_cast<const volatile uint8_t*>(src + i) : __ldg(src + i);
        if (DST) dst[i] = b;
        if (CRC) r = t0[(r ^ b) & 0xffu] ^ (r >> 8);
    }
    return r;
}

__device__ __forceinline__ uint32_t find_piece(const uint32_t* prefix, uint32_t n, uint32_t u) {
    uint32_t lo = 0, hi = n;  // largest p in [0,n) with prefix[p] <= u
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(prefix + mid) <= u)
            lo = mid;
        else
            hi = mid;
    }
    return lo;
}

template <bool DST>
__global__ void expand_units_kernel(const Piece* __restrict__ pieces, uint32_t n_pieces, const uint32_t* __restrict__ prefix,
                                    uint32_t seg_shift, Unit* __restrict__ units, uint32_t cap) {
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= min(__ldg(prefix + n_pieces), cap)) return;
    const uint32_t p = find_piece(prefix, n_pieces, u);
    const Piece pc = pieces[p];
    const Geom g = piece_geom<DST>(pc, seg_shift);
    const uint32_t s = u - __ldg(prefix + p);
    const uint64_t seg_off = uint64_t(s) << seg_shift;
    Unit un;
    un.L = 0;
    if (s < g.nseg) {
        const uint64_t rem = g.body - seg_off;
        un.L = rem < (1ull << seg_shift) ? static_cast<uint32_t>(rem) : (1u << seg_shift);
    }
    un.src = pc.src + g.head + seg_off;
    un.dst = DST ? pc.dst + g.head + seg_off : nullptr;
    un.piece = p;
    un.head = s == 0 ? g.head : 0u;
    un.tail = s + 1 == g.units ? g.tail : 0u;
    units[u] = un;
}

__device__ __forceinline__ Unit ld_unit(const Unit* p) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(p)), b = __ldg(reinterpret_cast<const uint4*>(p) + 1);
    Unit un;
    un.src = reinterpret_cast<const uint8_t*>(uint64_t(a.x) | (uint64_t(a.y) << 32));
    un.dst = reinterpret_cast<uint8_t*>(uint64_t(a.z) | (uint64_t(a.w) << 32));
    un.L = b.x, un.piece = b.y, un.head = b.z, un.tail = b.w;
    return un;
}

template <bool CRC, bool DST, int T>
__global__ void __launch_bounds__(1024, 1)
    walk_kernel(const Unit* __restrict__ units, const uint32_t* __restrict__ total_units, const CrcConsts* __restrict__ cc,
                uint32_t* __restrict__ partial, uint32_t partial_cap, uint32_t* __restrict__ headraw, uint32_t* __restrict__ tailraw) {
    extern __shared__ uint32_t smem[];
    const uint32_t total = min(__ldg(total_units), partial_cap);
    const uint32_t per = (total + gridDim.x - 1) / gridDim.x;
    const uint32_t u0 = min(total, blockIdx.x * per), u1 = min(total, u0 + per);
    if (u0 >= u1) return;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t poly = 0;
    if (CRC) {
        const uint32_t* m = &cc->m[0][0];
        for (uint32_t i = tid; i < kTmWords; i += 1024) smem[i] = __ldg(m + (i >> 5));
        if (tid < 256) smem[kTmWords + tid] = cc->t0[tid];
        if (tid < 64) smem[kTmWords + 256 + tid] = cc->xp128[tid];
        if (tid < 16) smem[kTmWords + 256 + 64 + tid] = cc->pw8[tid];
        poly = cc->poly;
        __syncthreads();
    }
    const uint32_t* t0 = smem + kTmWords;
    if (u0 + warp >= u1) return;
    Unit cur = ld_unit(units + u0 + warp);
    for (uint32_t u = u0 + warp; u < u1; u += 32) {
        const Unit nxt = ld_unit(units + (u + 32 < u1 ? u + 32 : u));  // next unit's record travels behind this walk
        const uint32_t raw = walk_segment<CRC, DST, T>(cur.src, cur.dst, cur.L, lane, smem, poly);
        if (CRC && lane == 0) partial[u] = raw;
        if (cur.head && lane == 1) {
            const uint32_t r = walk_bytes<CRC, DST>(cur.src - cur.head, DST ? cur.dst - cur.head : nullptr, cur.head, t0);
            if (CRC) headraw[cur.piece] = r;
        }
        if (cur.tail && lane == 2) {
            const uint32_t r = walk_bytes<CRC, DST>(cur.src + cur.L, DST ? cur.dst + cur.L : nullptr, cur.tail, t0);
            if (CRC) tailraw[cur.piece] = r;
        }
        cur = nxt;
    }
}

// Fold unit partials into one CRC per block.  One WARP per block: the block's units [prefix[p0], prefix[p1]) are cut into
// 32 contiguous lane ranges; every lane runs the Horner recurrence acc <- acc * x^(8*len_u) (+) raw_u over its range while
// also accumulating the product of the multipliers, then (acc, mult) pairs are combined across lanes with a shuffle tree
// ((a1,m1) o (a2,m2) = (a1*m2 + a2, m1*m2)).  Start value 0xFFFFFFFF and final complement make the result bit-identical
// to crc32fast / zlib (or CRC-32C).  first/last == nullptr: block b is piece b.
template <bool DST>
__global__ void __launch_bounds__(256)
    fold_blocks_kernel(const Piece* __restrict__ pieces, const uint32_t* __restrict__ prefix, const uint32_t* __restrict__ first,
                       const uint32_t* __restrict__ last, uint32_t n_blocks, uint32_t n_pieces, uint32_t seg_shift, uint32_t xp_seg,
                       const CrcConsts* __restrict__ cc, const uint32_t* __restrict__ partial, const uint32_t* __restrict__ headraw,
                       const uint32_t* __restrict__ tailraw, uint32_t* __restrict__ out) {
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= n_blocks) return;
    const uint32_t poly = cc->poly;
    const uint32_t p0 = first ? first[b] : b, p1 = first ? last[b] : b + 1;
    uint32_t acc = 0, mult = kOne;
    if (p1 > p0) {
        const uint32_t u0 = prefix[p0], u1 = prefix[p1];
        const uint32_t per = (u1 - u0 + 31) / 32;
        const uint32_t ua = min(u1, u0 + lane * per), ub = min(u1, ua + per);
        if (ua < ub) {
            uint32_t p = find_piece(prefix, n_pieces, ua);
            for (uint32_t u = ua; u < ub; u++) {
                while (u >= prefix[p + 1]) p++;
                const Piece pc = pieces[p];
                const Geom g = piece_geom<DST>(pc, seg_shift);
                const uint32_t s = u - prefix[p];
                if (s == 0 && g.head) {
                    const uint32_t m = cc->pw8[g.head];
                    acc = gf_mul(acc, m, poly) ^ headraw[p], mult = gf_mul(mult, m, poly);
                }
                if (s < g.nseg) {
                    const uint64_t rem = g.body - (uint64_t(s) << seg_shift);
                    const uint32_t m = rem >= (1ull << seg_shift) ? xp_seg : gf_xpow(8 * rem, poly);
                    acc = gf_mul(acc, m, poly) ^ partial[u], mult = gf_mul(mult, m, poly);
                }
                if (s + 1 == g.units && g.tail) {
                    const uint32_t m = cc->pw8[g.tail];
                    acc = gf_mul(acc, m, poly) ^ tailraw[p], mult = gf_mul(mult, m, poly);
                }
            }
        }
    }
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t a2 = __shfl_down_sync(0xffffffffu, acc, d), m2 = __shfl_down_sync(0xffffffffu, mult, d);
        if ((lane & (2 * d - 1)) == 0) {
            acc = gf_mul(acc, m2, poly) ^ a2;
            mult = gf_mul(mult, m2, poly);
        }
    }
    if (lane == 0) out[b] = ~(gf_mul(0xffffffffu, mult, poly) ^ acc);
}

// ------------------------------------------------------------------ small inputs: one launch instead of a launch train
//
// A FUSE-sized read (config C5: 256 KiB files) is latency-bound: the five launches of the walker train (prep, scan, expand, walk,
// fold) and the 128 KB table replication cost more than the work.  For <= ~1 MiB in total, ONE kernel does a block per CTA:
//   * slicing-by-4 tables (4 KB) are built in shared memory from the byte table;
//   * the block is cut into 1024 chunks of S bytes, RIGHT-aligned (thread 1023 owns the last S bytes; the first chunk may be short
//     or empty -- leading zeros do not change a raw CRC), each thread runs a plain table CRC over its chunk;
//   * init 0xFFFFFFFF is folded into the data (the first four message bytes are complemented), so no x^(8*len) is needed;
//   * chunk CRCs combine pairwise, crc(A||B) = crc(A) * x^(8|B|) + crc(B) with |B| = S * 2^k at level k: the multiplier is squared
//     from level to level, starting at x^(8S) = xp128[S/16].
constexpr uint32_t kSmallMaxBlock = 1024u * 1008u;  // S <= 1008 so that S/16 < 64 (xp128 table)

__global__ void __launch_bounds__(1024) crc_small_kernel(const uint8_t* __restrict__ base, const uint64_t* __restrict__ off, const uint64_t* __restrict__ len,
                                                         const CrcConsts* __restrict__ cc, uint32_t* __restrict__ out) {
    __shared__ uint32_t T[4][256];
    __shared__ uint32_t part[32];
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5, b = blockIdx.x;
    const uint8_t* src = base + off[b];
    const uint32_t n = static_cast<uint32_t>(len[b]);
    if (t < 256) T[0][t] = cc->t0[t];
    __syncthreads();
#pragma unroll
    for (int k = 1; k < 4; k++) {
        if (t < 256) T[k][t] = (T[k - 1][t] >> 8) ^ T[0][T[k - 1][t] & 0xffu];
        __syncthreads();
    }
    if (n < 4) {  // the init cannot be folded into fewer than four bytes: the plain definition, one thread
        if (t == 0) {
            uint32_t c = 0xffffffffu;
            for (uint32_t i = 0; i < n; i++) c = T[0][(c ^ __ldg(src + i)) & 0xffu] ^ (c >> 8);
            out[b] = n ? ~c : 0u;
        }
        return;
    }
    const uint32_t S = ((n + 1023u) / 1024u + 15u) & ~15u;
    const int64_t end = int64_t(n) - int64_t(1023u - t) * S;
    const int64_t beg = end - S;
    uint32_t c = 0;
    if (end > 0) {
        uint32_t i = beg > 0 ? uint32_t(beg) : 0u;
        const uint32_t e = uint32_t(end);
        // message bytes 0..3 carry the folded init; then bytes up to a 4-byte aligned ADDRESS; then words; then the tail
        for (; i < e && (i < 4 || ((reinterpret_cast<uintptr_t>(src) + i) & 3u)); i++) c = T[0][(c ^ __ldg(src + i) ^ (i < 4 ? 0xffu : 0u)) & 0xffu] ^ (c >> 8);
        for (; i + 4 <= e; i += 4) {
            c ^= __ldg(reinterpret_cast<const uint32_t*>(src + i));
            c = T[3][c & 0xffu] ^ T[2][(c >> 8) & 0xffu] ^ T[1][(c >> 16) & 0xffu] ^ T[0][c >> 24];
        }
        for (; i < e; i++) c = T[0][(c ^ __ldg(src + i)) & 0xffu] ^ (c >> 8);
    }
    const uint32_t poly = cc->poly;
    uint32_t m = cc->xp128[S >> 4];  // x^(8S)
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {  // lanes: (left, right) pairs, the right one is d lanes up
        const uint32_t right = __shfl_down_sync(0xffffffffu, c, d);
        if ((lane & (2 * d - 1)) == 0) c = gf_mul(c, m, poly) ^ right;
        m = gf_mul(m, m, poly);
    }
    if (lane == 0) part[warp] = c;
    __syncthreads();
    if (warp == 0) {
        c = part[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t right = __shfl_down_sync(0xffffffffu, c, d);
            if ((lane & (2 * d - 1)) == 0) c = gf_mul(c, m, poly) ^ right;
            m = gf_mul(m, m, poly);
        }
        if (lane == 0) out[b] = ~c;
    }
}

// K3 for small inputs: a CTA per segment, 16 bytes per thread and step; vector accesses when both sides are 16-byte aligned.
__global__ void __launch_bounds__(256) gather_small_kernel(const uint8_t* __restrict__ src, const CvSeg* __restrict__ segs, uint8_t* __restrict__ dst) {
    const CvSeg sg = segs[blockIdx.x];
    const uint8_t* s = src + sg.src_off;
    uint8_t* d = dst + sg.dst_off;
    const uint64_t n = sg.len;
    if (((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d)) & 15u) == 0) {
        const uint64_t nv = n >> 4;
        for (uint64_t i = threadIdx.x; i < nv; i += blockDim.x) st_vec(reinterpret_cast<uint4*>(d) + i, ld_plain(reinterpret_cast<const uint4*>(s) + i));
        for (uint64_t i = (nv << 4) + threadIdx.x; i < n; i += blockDim.x) d[i] = s[i];
    } else if (((reinterpret_cast<uintptr_t>(s) ^ reinterpret_cast<uintptr_t>(d)) & 3u) == 0) {  // same phase: words after a byte head
        const uint32_t head = static_cast<uint32_t>((4u - (reinterpret_cast<uintptr_t>(d) & 3u)) & 3u);
        const uint64_t h = head < n ? head : n;
        if (threadIdx.x < h) d[threadIdx.x] = s[threadIdx.x];
        const uint64_t nw = (n - h) >> 2;
        for (uint64_t i = threadIdx.x; i < nw; i += blockDim.x) reinterpret_cast<uint32_t*>(d + h)[i] = __ldg(reinterpret_cast<const uint32_t*>(s + h) + i);
        for (uint64_t i = h + (nw << 2) + threadIdx.x; i < n; i += blockDim.x) d[i] = s[i];
    } else {
        for (uint64_t i = threadIdx.x; i < n; i += blockDim.x) d[i] = __ldg(s + i);
    }
}

__global__ void verify_crcs_kernel(const uint32_t* crc, const uint32_t* expect, const uint8_t* skip, uint32_t n, uint32_t* n_bad,
                                   uint8_t* bad_mask) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool bad = i < n && !(skip && skip[i]) && crc[i] != expect[i];
    if (i < n && bad_mask) bad_mask[i] = bad;
    const uint32_t m = __ballot_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(n_bad, __popc(m));
}

// ------------------------------------------------------------------ K5: gather with a dtype conversion
// The conversions are integer arithmetic on the bit patterns (no FP state, no intrinsics), IEEE round-to-nearest-even.

__device__ __forceinline__ uint32_t f16_to_f32(uint32_t h) {  // exact
    const uint32_t sign = (h & 0x8000u) << 16, e = (h >> 10) & 0x1fu;
    uint32_t m = h & 0x3ffu;
    if (e == 0x1fu) return sign | 0x7f800000u | (m << 13);  // inf, NaN (payload kept)
    if (e) return sign | ((e + 112u) << 23) | (m << 13);
    if (!m) return sign;
    uint32_t k = 0;  // subnormal m * 2^-24: normalise, 2^(-14-k) with k the shifts that bring the top bit to bit 10
    while (!(m & 0x400u)) m <<= 1, k++;
    return sign | ((113u - k) << 23) | ((m & 0x3ffu) << 13);
}

__device__ __forceinline__ uint32_t f32_to_f16(uint32_t u) {
    const uint32_t sign = (u >> 16) & 0x8000u, a = u & 0x7fffffffu;
    if (a > 0x7f800000u) return sign | 0x7e00u;  // NaN
    if (a >= 0x477ff000u) return sign | 0x7c00u;  // |x| >= 65520 (halfway above the largest half, 65504): inf
    if (a >= 0x38800000u) {                       // normal half: rebias the exponent, round the 13 dropped bits
        const uint32_t h = (a - 0x38000000u) >> 13, r = a & 0x1fffu;
        return sign | (h + (r > 0x1000u || (r == 0x1000u && (h & 1u))));
    }
    if (a <= 0x33000000u) return sign;  // |x| <= 2^-25, half the smallest subnormal: ties to the even zero
    const uint32_t s = 126u - (a >> 23), m = (a & 0x7fffffu) | 0x800000u;  // subnormal half: x / 2^-24 = m >> s, s in [14, 24]
    const uint32_t h = m >> s, r = m & ((1u << s) - 1u), half = 1u << (s - 1u);
    return sign | (h + (r > half || (r == half && (h & 1u))));  // a carry into bit 10 is the smallest normal: still right
}

__device__ __forceinline__ uint32_t f32_to_bf16(uint32_t u) {
    if ((u & 0x7fffffffu) > 0x7f800000u) return (u >> 16) | 0x40u;  // NaN: quiet, sign and top payload bits kept
    return (u + 0x7fffu + ((u >> 16) & 1u)) >> 16;                  // overflow carries into the exponent: inf
}

__device__ __forceinline__ uint32_t cast_size(int32_t dt) { return dt == CV_DTYPE_F32 ? 4u : 2u; }

__device__ __forceinline__ uint32_t cast_elem(uint32_t v, int32_t sdt, int32_t ddt) {
    if (sdt == ddt) return v;
    const uint32_t f = sdt == CV_DTYPE_F16 ? f16_to_f32(v) : sdt == CV_DTYPE_BF16 ? v << 16 : v;
    return ddt == CV_DTYPE_F16 ? f32_to_f16(f) : ddt == CV_DTYPE_BF16 ? f32_to_bf16(f) : f;
}

__device__ __forceinline__ uint32_t ld_elem(const uint8_t* p, uint32_t size) {
    return size == 4 ? *reinterpret_cast<const uint32_t*>(p) : *reinterpret_cast<const uint16_t*>(p);
}

__device__ __forceinline__ void st_elem(uint8_t* p, uint32_t size, uint32_t v) {
    if (size == 4) *reinterpret_cast<uint32_t*>(p) = v;
    else *reinterpret_cast<uint16_t*>(p) = static_cast<uint16_t>(v);
}

// 8 source elements from p (aligned to the element size only), in the widest loads the address allows
__device__ __forceinline__ void ld_chunk(const uint8_t* p, uint32_t size, uint32_t v[8]) {
    const uint32_t a = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(p)) & 15u;
    if (size == 4 && a == 0) {
        const uint4 x = ld_plain(reinterpret_cast<const uint4*>(p)), y = ld_plain(reinterpret_cast<const uint4*>(p + 16));
        v[0] = x.x, v[1] = x.y, v[2] = x.z, v[3] = x.w, v[4] = y.x, v[5] = y.y, v[6] = y.z, v[7] = y.w;
    } else if (size == 4 && (a & 7u) == 0) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint64_t w = reinterpret_cast<const uint64_t*>(p)[k];
            v[2 * k] = static_cast<uint32_t>(w), v[2 * k + 1] = static_cast<uint32_t>(w >> 32);
        }
    } else if (size == 2 && a == 0) {
        const uint4 x = ld_plain(reinterpret_cast<const uint4*>(p));
        const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int k = 0; k < 4; k++) v[2 * k] = w[k] & 0xffffu, v[2 * k + 1] = w[k] >> 16;
    } else if (size == 2 && (a & 3u) == 0) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t w = reinterpret_cast<const uint32_t*>(p)[k];
            v[2 * k] = w & 0xffffu, v[2 * k + 1] = w >> 16;
        }
    } else {
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = ld_elem(p + k * size, size);
    }
}

// ---- the scaled instance's additions: FP8 sources and a scale per element
// The FP8 decoders are branch-free (selects, no normalisation loop): a warp's 8 x 32 elements mix subnormals with normals.

__device__ __forceinline__ uint32_t small_to_f32(uint32_t m) {  // F32 bits of the integer m < 2^24: exact
#if defined(__CUDA_ARCH__)
    return __float_as_uint(__uint2float_rn(m));
#else
    const float x = static_cast<float>(m);
    memcpy(&m, &x, 4);
    return m;
#endif
}

__device__ __forceinline__ uint32_t e4m3_to_f32(uint32_t b) {  // exact; no infinities, 0x7f / 0xff are NaN
    const uint32_t sign = (b & 0x80u) << 24, a = b & 0x7fu;
    if (a == 0x7fu) return sign | 0x7fc00000u;
    // normal: exponent e + 120, mantissa m, i.e. (a + (120 << 3)) << 20; subnormal m * 2^-9: the float m with 9 off its exponent
    return sign | (a >= 8u ? (a + 0x3c0u) << 20 : a ? small_to_f32(a) - (9u << 23) : 0u);
}

__device__ __forceinline__ uint32_t e5m2_to_f32(uint32_t b) {  // exact; the top byte of an F16
    const uint32_t sign = (b & 0x80u) << 24, a = b & 0x7fu;
    if (a >= 0x7cu) return sign | 0x7f800000u | ((a & 3u) << 21);  // inf, NaN (payload kept)
    // normal: exponent e + 112, i.e. (a + (112 << 2)) << 21; subnormal m * 2^-16
    return sign | (a >= 4u ? (a + 0x1c0u) << 21 : a ? small_to_f32(a) - (16u << 23) : 0u);
}

__device__ __forceinline__ bool is_f8(int32_t dt) { return dt == CV_DTYPE_F8_E4M3 || dt == CV_DTYPE_F8_E5M2; }

// any source element -> F32 bits, exact
__device__ __forceinline__ uint32_t to_f32(uint32_t v, int32_t sdt) {
    return sdt == CV_DTYPE_F8_E4M3 ? e4m3_to_f32(v) : sdt == CV_DTYPE_F8_E5M2 ? e5m2_to_f32(v) : sdt == CV_DTYPE_F16 ? f16_to_f32(v)
         : sdt == CV_DTYPE_BF16 ? v << 16 : v;
}

__device__ __forceinline__ uint32_t from_f32(uint32_t f, int32_t ddt) {
    return ddt == CV_DTYPE_F16 ? f32_to_f16(f) : ddt == CV_DTYPE_BF16 ? f32_to_bf16(f) : f;
}

// one IEEE F32 multiply, round-to-nearest-even, never contracted into an FMA
__device__ __forceinline__ uint32_t f32_mul(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(__fmul_rn(__uint_as_float(a), __uint_as_float(b)));
#else
    float x, y;
    memcpy(&x, &a, 4), memcpy(&y, &b, 4);
    x *= y;
    memcpy(&a, &x, 4);
    return a;
#endif
}

// 8 FP8 elements from p: one 8-byte load when p is 8-byte aligned, bytes otherwise
__device__ __forceinline__ void ld_chunk8(const uint8_t* p, uint32_t v[8]) {
    if ((reinterpret_cast<uintptr_t>(p) & 7u) == 0) {
        const uint64_t w = *reinterpret_cast<const uint64_t*>(p);
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = static_cast<uint32_t>(w >> (8 * k)) & 0xffu;
    } else {
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = p[k];
    }
}

// a / b, in 32 bits when both fit (every tensor below 2^32 elements): the 64-bit division is a long software sequence
__device__ __forceinline__ uint64_t udiv(uint64_t a, uint64_t b) { return (a | b) >> 32 ? a / b : uint64_t(uint32_t(a) / uint32_t(b)); }

// The scale of the element in hand, kept in a register and stepped element by element: (i, j) is the element's view position, as
// (ib, ir) = divmod(i, block_rows) and (jb, jr) = divmod(j, block_cols).  Found by division once per chunk (start), then only
// compared and incremented; the scale is reloaded when the element enters another tile.  No scale table entry: s = 1.0 (exact).
// step() moves to the NEXT element and loads its scale, so it is called only when that element exists (before every element but the
// first): stepping past the range's last element could address a scale beyond the caller's buffer (the last view row of a per-tensor,
// per-row or whole-tile grid wraps into scale row scale_rows).
struct ScaleWalk {
    const uint8_t* p;
    int32_t dt;
    uint64_t cols, br, bc, scols, j, jr, jb, ir, ib;
    uint32_t s;
    __device__ __forceinline__ void load() {
        const uint64_t q = ib * scols + jb;
        s = dt == CV_DTYPE_F32 ? __ldg(reinterpret_cast<const uint32_t*>(p) + q)
          : dt == CV_DTYPE_F16 ? f16_to_f32(__ldg(reinterpret_cast<const uint16_t*>(p) + q))
                               : uint32_t(__ldg(reinterpret_cast<const uint16_t*>(p) + q)) << 16;
    }
    __device__ __forceinline__ void start(const CvScaleSeg& g, uint64_t row, uint64_t e) {
        p = static_cast<const uint8_t*>(g.scale);
        s = 0x3f800000u;
        if (!p) return;
        dt = g.scale_dtype, cols = g.cols, br = g.block_rows, bc = g.block_cols, scols = g.scale_cols;
        const uint64_t v = g.view0 + row * g.view_step + e, i = udiv(v, cols);
        j = v - i * cols, ib = udiv(i, br), ir = i - ib * br, jb = udiv(j, bc), jr = j - jb * bc;
        load();
    }
    __device__ __forceinline__ bool flat(uint32_t m) const { return !p || (jr + m <= bc && j + m <= cols); }  // the next m share s
    __device__ __forceinline__ void step() {
        if (!p) return;
        if (++j == cols) {
            j = jr = jb = 0;
            if (++ir == br) ir = 0, ib++;
            load();
        } else if (++jr == bc) {
            jr = 0, jb++;
            load();
        }
    }
};

// A whole chunk through F32 with its scales.  Called with constant dtypes for the FP8 pairs (scale_chunk), so each pair inlines to
// straight-line code with no per-element dtype selects.
__device__ __forceinline__ void scale8(uint32_t v[8], int32_t sdt, int32_t ddt, ScaleWalk& w) {
    if (w.flat(8)) {  // one scale for the chunk
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = from_f32(f32_mul(to_f32(v[j], sdt), w.s), ddt);
    } else {  // the chunk crosses a tile edge or a view row
#pragma unroll
        for (int j = 0; j < 8; j++) {
            if (j) w.step();
            v[j] = from_f32(f32_mul(to_f32(v[j], sdt), w.s), ddt);
        }
    }
}

__device__ __forceinline__ void scale_chunk(uint32_t v[8], int32_t sdt, int32_t ddt, ScaleWalk& w) {
    if (sdt == CV_DTYPE_F8_E4M3 && ddt == CV_DTYPE_BF16) scale8(v, CV_DTYPE_F8_E4M3, CV_DTYPE_BF16, w);
    else if (sdt == CV_DTYPE_F8_E4M3 && ddt == CV_DTYPE_F16) scale8(v, CV_DTYPE_F8_E4M3, CV_DTYPE_F16, w);
    else if (sdt == CV_DTYPE_F8_E4M3) scale8(v, CV_DTYPE_F8_E4M3, CV_DTYPE_F32, w);
    else if (sdt == CV_DTYPE_F8_E5M2 && ddt == CV_DTYPE_BF16) scale8(v, CV_DTYPE_F8_E5M2, CV_DTYPE_BF16, w);
    else if (sdt == CV_DTYPE_F8_E5M2 && ddt == CV_DTYPE_F16) scale8(v, CV_DTYPE_F8_E5M2, CV_DTYPE_F16, w);
    else if (sdt == CV_DTYPE_F8_E5M2) scale8(v, CV_DTYPE_F8_E5M2, CV_DTYPE_F32, w);
    else scale8(v, sdt, ddt, w);  // a scaled F32 / F16 / BF16 segment
}

// Grid-stride over the work chunks of all segments (CvCastSeg::first numbers them): neighbouring threads take neighbouring chunks, so
// every load and store of a warp is coalesced whatever the shape.  In a row whose destination is `head` elements short of a 16-byte
// boundary, chunk 0 holds those head elements and chunk k >= 1 the 8 elements from head + 8(k-1) on (with head = 0, chunk k holds 8k..):
// every whole chunk stores one (2-byte destination) or two (4-byte destination) aligned 16-byte vectors.
// SCALED (cvk_gather_cast_scaled) adds FP8 sources and scales[]; the plain instance never reads `scales` and compiles to the code it
// compiled to before the scaled one existed.
template <bool SCALED>
__global__ void __launch_bounds__(256) gather_cast_kernel(const uint8_t* __restrict__ src, const CvCastSeg* __restrict__ segs, uint32_t n,
                                                          uint8_t* __restrict__ dst, const CvScaleSeg* __restrict__ scales) {
    const uint64_t total = segs[n - 1].first + segs[n - 1].rows * CV_CAST_ROW_CHUNKS(segs[n - 1].elems);
    uint32_t d = 0;  // the segment of the previous chunk: chunks only grow, so the search starts there
    for (uint64_t c = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; c < total; c += uint64_t(gridDim.x) * blockDim.x) {
        if (d + 1 < n && segs[d + 1].first <= c) {  // the last segment whose first chunk is <= c (empty segments share their first)
            uint32_t lo = d + 1, hi = n - 1;
            while (lo < hi) {
                const uint32_t mid = (lo + hi + 1) >> 1;
                if (segs[mid].first <= c) lo = mid;
                else hi = mid - 1;
            }
            d = lo;
        }
        const CvCastSeg& s = segs[d];
        const uint64_t cpr = CV_CAST_ROW_CHUNKS(s.elems), rel = c - s.first;
        if (c < s.first || rel >= s.rows * cpr) continue;  // a table whose `first` leaves gaps: nothing is written outside a row
        const int32_t sdt = s.src_dtype, ddt = s.dst_dtype;
        const bool f8 = SCALED && is_f8(sdt);
        if ((!f8 && sdt != CV_DTYPE_F32 && sdt != CV_DTYPE_F16 && sdt != CV_DTYPE_BF16) ||
            (ddt != CV_DTYPE_F32 && ddt != CV_DTYPE_F16 && ddt != CV_DTYPE_BF16))
            continue;
        // through F32 with a multiply: FP8 sources and scaled segments (the scale is 1.0 for an unscaled FP8 one)
        const bool mul = SCALED && (f8 || scales[d].scale);
        const uint32_t ss = f8 ? 1u : cast_size(sdt), ds = cast_size(ddt);
        const uint64_t row = rel < cpr ? 0 : rel / cpr, k = rel - row * cpr;
        const uint8_t* sp = src + s.src_off + row * s.src_pitch;
        uint8_t* dp = dst + s.dst_off + row * s.dst_pitch;
        const uint32_t head = ((16u - (static_cast<uint32_t>(reinterpret_cast<uintptr_t>(dp)) & 15u)) & 15u) / ds;
        const int64_t e0 = 8 * int64_t(k) - int64_t((8u - head) & 7u);  // chunk k: elements [e0, e0 + 8) of the row, clipped to it
        const int64_t lo = e0 > 0 ? e0 : 0, hi = e0 + 8 < int64_t(s.elems) ? e0 + 8 : int64_t(s.elems);
        if (lo >= hi) continue;
        ScaleWalk w;
        if (mul) w.start(scales[d], row, uint64_t(lo));
        if (hi - lo == 8) {  // a whole chunk: its destination is 16-byte aligned
            uint32_t v[8];
            if (f8) ld_chunk8(sp + lo, v);
            else ld_chunk(sp + lo * ss, ss, v);
            if (!mul) {
#pragma unroll
                for (int j = 0; j < 8; j++) v[j] = cast_elem(v[j], sdt, ddt);
            } else {
                scale_chunk(v, sdt, ddt, w);
            }
            uint4* o = reinterpret_cast<uint4*>(dp + lo * ds);
            if (ds == 2) {
                st_vec(o, make_uint4(v[0] | v[1] << 16, v[2] | v[3] << 16, v[4] | v[5] << 16, v[6] | v[7] << 16));
            } else {
                st_vec(o, make_uint4(v[0], v[1], v[2], v[3]));
                st_vec(o + 1, make_uint4(v[4], v[5], v[6], v[7]));
            }
        } else if (!mul) {
            for (int64_t e = lo; e < hi; e++) st_elem(dp + e * ds, ds, cast_elem(ld_elem(sp + e * ss, ss), sdt, ddt));
        } else {
            for (int64_t e = lo; e < hi; e++) {
                if (e > lo) w.step();
                const uint32_t x = f8 ? uint32_t(sp[e]) : ld_elem(sp + e * ss, ss);
                st_elem(dp + e * ds, ds, from_f32(f32_mul(to_f32(x, sdt), w.s), ddt));
            }
        }
    }
}

// ------------------------------------------------------------------ host side

static std::atomic<uint64_t> g_launches{0};
static std::mutex g_mu;
constexpr int kMaxDev = 16;
static CrcConsts* g_consts[kMaxDev][2];
static int g_sm_count[kMaxDev];
static cudaMemPool_t g_pool[kMaxDev];  // workspace pool that keeps its memory across synchronisation points
static bool g_ready[kMaxDev];

#define CV_TRY(x)                             \
    do {                                      \
        cudaError_t e_ = (x);                 \
        if (e_ != cudaSuccess) return int(e_); \
    } while (0)

// Launch on the device that owns the data, whatever the calling thread's current device is (a host that links
// its own CUDA runtime -- torch, a Rust crate -- may not share "current device" state with this library).
struct DeviceGuard {
    int prev = -1, dev = -1;
    bool switched = false;
    explicit DeviceGuard(const void* device_ptr) {
        cudaGetDevice(&prev);
        dev = prev;
        cudaPointerAttributes a;
        if (device_ptr && cudaPointerGetAttributes(&a, device_ptr) == cudaSuccess && a.type == cudaMemoryTypeDevice) dev = a.device;
        else cudaGetLastError();
        if (dev != prev) switched = cudaSetDevice(dev) == cudaSuccess;
    }
    ~DeviceGuard() {
        if (switched) cudaSetDevice(prev);
    }
};

static int ensure_device(int* dev_out) {
    int dev = 0;
    CV_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= kMaxDev) return int(cudaErrorInvalidDevice);
    *dev_out = dev;
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_ready[dev]) return 0;
    for (int pid = 0; pid < 2; pid++) {
        CrcConsts* h = new CrcConsts;
        build_consts(poly_of(pid), h);
        CrcConsts* d = nullptr;
        cudaError_t e = cudaMalloc(&d, sizeof(CrcConsts));
        if (e == cudaSuccess) e = cudaMemcpy(d, h, sizeof(CrcConsts), cudaMemcpyHostToDevice);
        delete h;
        if (e != cudaSuccess) return int(e);
        g_consts[dev][pid] = d;
    }
    CV_TRY(cudaDeviceGetAttribute(&g_sm_count[dev], cudaDevAttrMultiProcessorCount, dev));
    {
        // Per-launch workspaces come from a private stream-ordered pool with an unlimited release threshold.  The default
        // pool hands its memory back to the driver at every synchronisation point (threshold 0), so a caller that syncs
        // between calls (every verify batch does) would pay a fresh physical allocation in front of each launch train.
        cudaMemPoolProps props = {};
        props.allocType = cudaMemAllocationTypePinned;
        props.handleTypes = cudaMemHandleTypeNone;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = dev;
        CV_TRY(cudaMemPoolCreate(&g_pool[dev], &props));
        uint64_t keep = ~0ull;
        CV_TRY(cudaMemPoolSetAttribute(g_pool[dev], cudaMemPoolAttrReleaseThreshold, &keep));
    }
    CV_TRY(cudaFuncSetAttribute(walk_kernel<true, false, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    CV_TRY(cudaFuncSetAttribute(walk_kernel<true, true, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    g_ready[dev] = true;
    return 0;
}

static std::atomic<bool> g_small_path{true};  // cvk_tune(5, 0/1): single-launch kernels for inputs of at most ~1 MiB
static std::atomic<int> g_seg_shift_override{0};  // cvk_tune(4, s): segment size 2^s for every launcher (0 = chosen from the input size)
constexpr uint32_t kStridedTrainRows = 1u << 22;
static std::atomic<uint32_t> g_strided_train{kStridedTrainRows};  // cvk_tune(6, r): rows per train of cvk_gather_strided
static uint32_t pick_seg_shift(uint64_t total_bytes, int sm_count) {
    if (const int o = g_seg_shift_override.load(std::memory_order_relaxed)) return static_cast<uint32_t>(o);
    // ~16 units per warp keeps the contiguous per-CTA ranges balanced for big inputs; small inputs get 16 KiB segments
    // (4 KiB below 4 MiB) so the per-block fold stays short.  4 KiB..1 MiB.
    const uint64_t target = total_bytes / (uint64_t(sm_count) * 32 * 16 + 1);
    uint32_t s = total_bytes >= (4u << 20) ? 14 : 12;
    while (s < 20 && (1ull << s) < target) s++;
    return s;
}

struct Workspace {
    Piece* pieces;
    Unit* units;
    uint32_t *counts, *prefix, *headraw, *tailraw, *partial, *first, *last;
    uint32_t partial_cap;
    void* base;
};

static int ws_alloc(Workspace* w, int dev, uint32_t n_pieces, uint32_t n_blocks, uint64_t total_bytes, uint32_t seg_shift,
                    cudaStream_t st) {
    auto up = [](size_t x) { return (x + 255) & ~size_t(255); };
    const uint64_t cap64 = uint64_t(n_pieces) + (total_bytes >> seg_shift) + 1;
    w->partial_cap = cap64 > 0xfffffff0ull ? 0xfffffff0u : uint32_t(cap64);
    const size_t s_pieces = up(sizeof(Piece) * size_t(n_pieces));
    const size_t s_n = up(4 * (size_t(n_pieces) + 1));
    const size_t s_part = up(4 * size_t(w->partial_cap));
    const size_t s_blk = up(4 * (size_t(n_blocks) + 1));
    const size_t s_units = up(sizeof(Unit) * size_t(w->partial_cap));
    const size_t total = s_pieces + s_units + 4 * s_n + s_part + 2 * s_blk;
    CV_TRY(cudaMallocFromPoolAsync(&w->base, total, g_pool[dev], st));
    uint8_t* p = static_cast<uint8_t*>(w->base);
    w->pieces = reinterpret_cast<Piece*>(p), p += s_pieces;
    w->units = reinterpret_cast<Unit*>(p), p += s_units;
    w->counts = reinterpret_cast<uint32_t*>(p), p += s_n;
    w->prefix = reinterpret_cast<uint32_t*>(p), p += s_n;
    w->headraw = reinterpret_cast<uint32_t*>(p), p += s_n;
    w->tailraw = reinterpret_cast<uint32_t*>(p), p += s_n;
    w->partial = reinterpret_cast<uint32_t*>(p), p += s_part;
    w->first = reinterpret_cast<uint32_t*>(p), p += s_blk;
    w->last = reinterpret_cast<uint32_t*>(p);
    CV_TRY(cudaMemsetAsync(w->first, 0, 2 * s_blk, st));
    return 0;
}

// end of a launch train: report the first launch error (if any) and hand the workspace back to the pool either way
static int ws_finish(Workspace& w, cudaStream_t st) {
    const cudaError_t launch = cudaGetLastError();
    const cudaError_t freed = cudaFreeAsync(w.base, st);
    return int(launch != cudaSuccess ? launch : freed);
}

static inline uint32_t cdiv(uint64_t a, uint32_t b) { return uint32_t((a + b - 1) / b); }

// optional timing of the dominant (walk) kernel: events on the launching stream, summed by cvk_profile_collect
static std::atomic<bool> g_prof_on{false};
static std::mutex g_prof_mu;
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_events;
struct WalkTimer {
    cudaStream_t st;
    cudaEvent_t a = nullptr, b = nullptr;
    explicit WalkTimer(cudaStream_t s) : st(s) {
        if (!g_prof_on.load(std::memory_order_relaxed)) return;
        if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) {
            a = b = nullptr;
            return;
        }
        cudaEventRecord(a, st);
    }
    ~WalkTimer() {
        if (!a) return;
        cudaEventRecord(b, st);
        std::lock_guard<std::mutex> lk(g_prof_mu);
        g_prof_events.emplace_back(a, b);
    }
};
// exclusive prefix sum of w.counts[0..n) into w.prefix[0..n]; headraw is free until the walker runs and holds the tile sums
static int launch_scan(const Workspace& w, uint32_t n, cudaStream_t st) {
    if (n <= 16384) {
        scan_counts_kernel<<<1, 1024, 0, st>>>(w.counts, n, w.prefix);
        return 1;
    }
    const uint32_t tiles = cdiv(n, 4096);
    tile_sums_kernel<<<tiles, 1024, 0, st>>>(w.counts, n, w.headraw);
    scan_tiles_kernel<<<tiles, 1024, 0, st>>>(w.counts, n, w.headraw, w.prefix);
    return 2;
}
#define CV_WALK_ARGS w.units, w.prefix + n, cc, w.partial, w.partial_cap, w.headraw, w.tailraw
// (pieces, prefix) -> one 32-byte record per unit; every walker launch is preceded by this
template <bool DST>
static void launch_expand(const Workspace& w, uint32_t n, uint32_t seg_shift, cudaStream_t st) {
    expand_units_kernel<DST><<<cdiv(w.partial_cap, 256), 256, 0, st>>>(w.pieces, n, w.prefix, seg_shift, w.units, w.partial_cap);
}

// Rows per tile of the DST walks: 4 for CRC+copy, 2 for copy-only (tools/kbench.py, DESIGN §3).
static void launch_walk_crc_dst(int dev, cudaStream_t st, const Workspace& w, uint32_t n, const CrcConsts* cc) {
    walk_kernel<true, true, 4><<<g_sm_count[dev], 1024, kSmemBytes, st>>>(CV_WALK_ARGS);
}

// copy-only walk: no shared memory, one CTA per SM (the kernels need > 32 registers, so two 1024-thread CTAs never fit).
// Sources may be another GPU's HBM mapped over NVLink (cvk_gather_shards_p2p): the DST walks use plain coherent loads only.
static void launch_walk_copy(int dev, cudaStream_t st, const Workspace& w, uint32_t n) {
    const CrcConsts* cc = nullptr;
    walk_kernel<false, true, 2><<<g_sm_count[dev], 1024, 0, st>>>(CV_WALK_ARGS);
}
#undef CV_WALK_ARGS
static inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

}  // namespace cv

using namespace cv;

extern "C" {

int cvk_init(int device) {
    int cur = 0;
    CV_TRY(cudaGetDevice(&cur));
    if (device != cur) CV_TRY(cudaSetDevice(device));
    int dev;
    const int rc = ensure_device(&dev);
    if (device != cur) cudaSetDevice(cur);
    return rc;
}

int cvk_tune(int what, int value) {
    if (what == 4 && (value == 0 || (value >= 12 && value <= 20))) g_seg_shift_override.store(value);
    else if (what == 5 && (value == 0 || value == 1)) g_small_path.store(value != 0);
    else if (what == 6 && value >= 0 && value <= int(kStridedTrainRows)) g_strided_train.store(value ? uint32_t(value) : kStridedTrainRows);
    else return int(cudaErrorInvalidValue);
    return 0;
}

uint64_t cvk_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int cvk_profile_enable(int on) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    for (auto& p : g_prof_events) cudaEventDestroy(p.first), cudaEventDestroy(p.second);
    g_prof_events.clear();
    g_prof_on.store(on != 0);
    return 0;
}

int cvk_profile_collect(double* walk_ms_total, uint32_t* walk_launches) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    double total = 0;
    uint32_t n = 0;
    for (auto& p : g_prof_events) {
        float ms = 0;
        cudaError_t e = cudaEventSynchronize(p.second);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, p.first, p.second);
        cudaEventDestroy(p.first), cudaEventDestroy(p.second);
        if (e != cudaSuccess) return int(e);
        total += ms, n++;
    }
    g_prof_events.clear();
    if (walk_ms_total) *walk_ms_total = total;
    if (walk_launches) *walk_launches = n;
    return 0;
}

int cvk_crc_blocks(const uint8_t* d_base, const uint64_t* d_off, const uint64_t* d_len, uint32_t n, int poly,
                   uint64_t total_bytes, uint32_t* d_crc_out, cv_stream_t stream) {
    if (n == 0) return 0;
    if (poly != 0 && poly != 1) return int(cudaErrorInvalidValue);
    DeviceGuard guard(d_crc_out);
    int dev;
    if (int rc = ensure_device(&dev)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (total_bytes <= kSmallMaxBlock && n <= 65535 && g_small_path.load(std::memory_order_relaxed)) {  // latency path: one launch, no workspace
        crc_small_kernel<<<n, 1024, 0, st>>>(d_base, d_off, d_len, g_consts[dev][poly], d_crc_out);
        count_launch();
        return int(cudaGetLastError());
    }
    const uint32_t seg_shift = pick_seg_shift(total_bytes, g_sm_count[dev]);
    Workspace w;
    if (int rc = ws_alloc(&w, dev, n, n, total_bytes, seg_shift, st)) return rc;
    const CrcConsts* cc = g_consts[dev][poly];
    prep_blocks_kernel<<<cdiv(n, 256), 256, 0, st>>>(d_base, d_off, d_len, n, seg_shift, w.pieces, w.counts);
    const int n_scan = launch_scan(w, n, st);
    launch_expand<false>(w, n, seg_shift, st);
    {
        WalkTimer wt(st);
        walk_kernel<true, false, 4><<<g_sm_count[dev], 1024, kSmemBytes, st>>>(w.units, w.prefix + n, cc, w.partial, w.partial_cap,
                                                                                       w.headraw, w.tailraw);
    }
    fold_blocks_kernel<false><<<cdiv(uint64_t(n) * 32, 256), 256, 0, st>>>(w.pieces, w.prefix, nullptr, nullptr, n, n, seg_shift,
                                                                           gf_xpow(8ull << seg_shift, poly_of(poly)), cc,
                                                                           w.partial, w.headraw, w.tailraw, d_crc_out);
    count_launch(4 + n_scan);
    return ws_finish(w, st);
}

int cvk_verify_crcs(const uint32_t* d_crc, const uint32_t* d_expect, uint32_t n, uint32_t* d_n_bad,
                    uint8_t* d_bad_mask, cv_stream_t stream) {
    return cvk_verify_crcs_masked(d_crc, d_expect, nullptr, n, d_n_bad, d_bad_mask, stream);
}

int cvk_verify_crcs_masked(const uint32_t* d_crc, const uint32_t* d_expect, const uint8_t* d_skip, uint32_t n, uint32_t* d_n_bad,
                           uint8_t* d_bad_mask, cv_stream_t stream) {
    if (n == 0) return 0;
    DeviceGuard guard(d_crc);
    verify_crcs_kernel<<<cdiv(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(d_crc, d_expect, d_skip, n, d_n_bad,
                                                                                   d_bad_mask);
    count_launch();
    return int(cudaGetLastError());
}

int cvk_expand_streams(const CvStreamDesc* d_streams, uint32_t n_streams, CvFrameDesc* d_desc_out, uint32_t n_frames,
                       cv_stream_t stream) {
    if (n_streams == 0) return 0;
    DeviceGuard guard(d_desc_out);
    expand_streams_kernel<<<cdiv(uint64_t(n_streams) * 32, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        d_streams, n_streams, d_desc_out, n_frames);
    count_launch();
    return int(cudaGetLastError());
}

static int frames_common(bool pack, const uint8_t* d_in, const CvFrameDesc* d_desc, uint32_t n_frames,
                         uint32_t n_blocks, uint8_t* d_out, int poly, uint64_t total_bytes, uint32_t* d_block_crc,
                         uint32_t* d_err_flags, cv_stream_t stream) {
    if (n_frames == 0) return 0;
    if (poly != 0 && poly != 1) return int(cudaErrorInvalidValue);
    DeviceGuard guard(d_out);
    int dev;
    if (int rc = ensure_device(&dev)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const uint32_t seg_shift = pick_seg_shift(total_bytes, g_sm_count[dev]);
    Workspace w;
    if (int rc = ws_alloc(&w, dev, n_frames, n_blocks, total_bytes, seg_shift, st)) return rc;
    const CrcConsts* cc = g_consts[dev][poly];
    if (pack)
        prep_pack_kernel<<<cdiv(n_frames, 256), 256, 0, st>>>(d_in, d_desc, n_frames, d_out, seg_shift, w.pieces,
                                                              w.counts);
    else
        prep_unpack_kernel<<<cdiv(n_frames, 256), 256, 0, st>>>(d_in, d_desc, n_frames, d_out, seg_shift, w.pieces,
                                                                w.counts, d_err_flags);
    const int n_scan = launch_scan(w, n_frames, st);
    launch_expand<true>(w, n_frames, seg_shift, st);
    count_launch(2 + n_scan);
    if (d_block_crc) {
        {
            WalkTimer wt(st);
            launch_walk_crc_dst(dev, st, w, n_frames, cc);
        }
        mark_block_ranges_kernel<<<cdiv(n_frames, 256), 256, 0, st>>>(d_desc, n_frames, n_blocks, w.first, w.last);
        fold_blocks_kernel<true><<<cdiv(uint64_t(n_blocks) * 32, 256), 256, 0, st>>>(
            w.pieces, w.prefix, w.first, w.last, n_blocks, n_frames, seg_shift, gf_xpow(8ull << seg_shift, poly_of(poly)), cc,
            w.partial, w.headraw, w.tailraw, d_block_crc);
        count_launch(3);
    } else {
        launch_walk_copy(dev, st, w, n_frames);
        count_launch();
    }
    return ws_finish(w, st);
}

int cvk_unpack_frames(const uint8_t* d_wire, const CvFrameDesc* d_desc, uint32_t n_frames, uint32_t n_blocks,
                      uint8_t* d_dst, int poly, uint64_t total_bytes, uint32_t* d_block_crc, uint32_t* d_err_flags,
                      cv_stream_t stream) {
    return frames_common(false, d_wire, d_desc, n_frames, n_blocks, d_dst, poly, total_bytes, d_block_crc,
                         d_err_flags, stream);
}

int cvk_pack_frames(const uint8_t* d_src, const CvFrameDesc* d_desc, uint32_t n_frames, uint32_t n_blocks,
                    uint8_t* d_wire, int poly, uint64_t total_bytes, uint32_t* d_block_crc, cv_stream_t stream) {
    return frames_common(true, d_src, d_desc, n_frames, n_blocks, d_wire, poly, total_bytes, d_block_crc, nullptr,
                         stream);
}

static int copy_pieces(Workspace& w, uint32_t n, uint32_t seg_shift, int dev, cudaStream_t st) {
    const int n_scan = launch_scan(w, n, st);
    launch_expand<true>(w, n, seg_shift, st);
    launch_walk_copy(dev, st, w, n);
    count_launch(2 + n_scan);
    return ws_finish(w, st);
}

int cvk_gather_pages(const uint8_t* d_src, const CvSeg* d_segs, uint32_t n, uint64_t total_bytes, uint8_t* d_dst,
                     cv_stream_t stream) {
    if (n == 0) return 0;
    DeviceGuard guard(d_dst);
    int dev;
    if (int rc = ensure_device(&dev)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (total_bytes <= (1u << 20) && n <= 4096 && g_small_path.load(std::memory_order_relaxed)) {  // latency path (a FUSE reply's pages): one launch
        gather_small_kernel<<<n, 256, 0, st>>>(d_src, d_segs, d_dst);
        count_launch();
        return int(cudaGetLastError());
    }
    const uint32_t seg_shift = pick_seg_shift(total_bytes, g_sm_count[dev]);
    Workspace w;
    if (int rc = ws_alloc(&w, dev, n, 0, total_bytes, seg_shift, st)) return rc;
    prep_segs_kernel<<<cdiv(n, 256), 256, 0, st>>>(d_src, d_segs, n, d_dst, seg_shift, w.pieces, w.counts);
    count_launch();
    return copy_pieces(w, n, seg_shift, dev, st);
}

int cvk_gather_strided(const uint8_t* d_src, const CvStridedSeg* d_segs, uint32_t n, uint64_t total_bytes, uint8_t* d_dst,
                       cv_stream_t stream) {
    if (n == 0) return 0;
    DeviceGuard guard(d_dst);
    int dev;
    if (int rc = ensure_device(&dev)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // the row numbering: descriptor d owns rows [pref[d], pref[d + 1]); a descriptor of empty rows owns none
    std::vector<CvStridedSeg> h(n);
    CV_TRY(cudaMemcpyAsync(h.data(), d_segs, sizeof(CvStridedSeg) * n, cudaMemcpyDeviceToHost, st));
    CV_TRY(cudaStreamSynchronize(st));
    std::vector<uint64_t> pref(size_t(n) + 1, 0);
    for (uint32_t d = 0; d < n; d++) pref[d + 1] = pref[d] + (h[d].len ? h[d].rows : 0);
    const uint64_t rows = pref[n];
    if (rows == 0) return 0;
    uint64_t* d_pref = nullptr;
    CV_TRY(cudaMallocFromPoolAsync(reinterpret_cast<void**>(&d_pref), sizeof(uint64_t) * pref.size(), g_pool[dev], st));
    cudaError_t ce = cudaMemcpyAsync(d_pref, pref.data(), sizeof(uint64_t) * pref.size(), cudaMemcpyHostToDevice, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);  // pref is this frame's (pageable) vector
    int rc = int(ce);
    const uint32_t seg_shift = pick_seg_shift(total_bytes, g_sm_count[dev]);
    const uint64_t train = g_strided_train.load(std::memory_order_relaxed);
    // one launch train per `train` rows: the workspace is bounded by the train, not by the row count
    for (uint64_t base = 0; base < rows && !rc; base += train) {
        const uint32_t cnt = uint32_t(rows - base < train ? rows - base : train);
        Workspace w;
        if ((rc = ws_alloc(&w, dev, cnt, 0, total_bytes, seg_shift, st))) break;
        prep_strided_kernel<<<cdiv(uint64_t(n) * 32, 256), 256, 0, st>>>(d_src, d_segs, d_pref, n, d_dst, base, cnt, seg_shift, w.pieces, w.counts);
        count_launch();
        rc = copy_pieces(w, cnt, seg_shift, dev, st);
    }
    const cudaError_t freed = cudaFreeAsync(d_pref, st);
    return rc ? rc : int(freed);
}

// K5, plain (d_scales == NULL) or scaled: one launch statement, the instance chosen through a function pointer
static int launch_cast(const uint8_t* d_src, const CvCastSeg* d_segs, const CvScaleSeg* d_scales, uint32_t n, uint64_t total_elems, uint8_t* d_dst,
                       cv_stream_t stream) {
    if (n == 0 || total_elems == 0) return 0;
    DeviceGuard guard(d_dst);
    int dev;
    if (int rc = ensure_device(&dev)) return rc;
    // the table stays on the device: the kernel takes the chunk count from its last entry.  One thread per 8 elements, at most 8
    // CTAs of 256 per SM; the grid-stride loop takes the rest (and the head chunks of many short rows).
    const uint64_t want = total_elems / (8 * 256) + 1, cap = uint64_t(g_sm_count[dev]) * 8;
    auto cast = d_scales ? gather_cast_kernel<true> : gather_cast_kernel<false>;
    cast<<<uint32_t(want < cap ? want : cap), 256, 0, static_cast<cudaStream_t>(stream)>>>(d_src, d_segs, n, d_dst, d_scales);
    count_launch();
    return int(cudaGetLastError());
}

int cvk_gather_cast(const uint8_t* d_src, const CvCastSeg* d_segs, uint32_t n, uint64_t total_elems, uint8_t* d_dst, cv_stream_t stream) {
    return launch_cast(d_src, d_segs, nullptr, n, total_elems, d_dst, stream);
}

int cvk_gather_cast_scaled(const uint8_t* d_src, const CvCastSeg* d_segs, const CvScaleSeg* d_scales, uint32_t n, uint64_t total_elems,
                           uint8_t* d_dst, cv_stream_t stream) {
    if (n && !d_scales) return int(cudaErrorInvalidValue);
    return launch_cast(d_src, d_segs, d_scales, n, total_elems, d_dst, stream);
}

int cvk_deinterleave_blocks(const uint8_t* d_gathered, uint64_t shard_stride, uint32_t world, uint64_t block_size,
                            uint64_t n_blocks, uint64_t file_len, uint8_t* d_dst, cv_stream_t stream) {
    if (n_blocks == 0) return 0;
    if (world == 0 || block_size == 0 || n_blocks > 0x7fffffffull) return int(cudaErrorInvalidValue);
    DeviceGuard guard(d_dst);
    int dev;
    if (int rc = ensure_device(&dev)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const uint32_t seg_shift = pick_seg_shift(file_len, g_sm_count[dev]);
    Workspace w;
    const uint32_t n = uint32_t(n_blocks);
    if (int rc = ws_alloc(&w, dev, n, 0, file_len, seg_shift, st)) return rc;
    prep_deinterleave_kernel<<<cdiv(n, 256), 256, 0, st>>>(d_gathered, shard_stride, world, block_size, n_blocks,
                                                           file_len, d_dst, seg_shift, w.pieces, w.counts);
    count_launch();
    return copy_pieces(w, n, seg_shift, dev, st);
}

int cvk_gather_shards_p2p(const uint8_t* const* shard_ptrs, uint32_t world, uint64_t block_size, uint64_t n_blocks, uint64_t file_len,
                          uint8_t* d_dst, cv_stream_t stream) {
    if (n_blocks == 0) return 0;
    if (world == 0 || world > 64 || block_size == 0 || n_blocks > 0x7fffffffull) return int(cudaErrorInvalidValue);
    DeviceGuard guard(d_dst);
    int dev;
    if (int rc = ensure_device(&dev)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const uint32_t seg_shift = pick_seg_shift(file_len, g_sm_count[dev]);
    Workspace w;
    const uint32_t n = uint32_t(n_blocks);
    if (int rc = ws_alloc(&w, dev, n, 64, file_len, seg_shift, st)) return rc;  // w.first doubles as the pointer table (>= 64*8 bytes)
    static_assert(sizeof(uint8_t*) == 8, "64-bit pointers");
    // kernels on this device read the peers' HBM directly: make sure peer access (this device -> owner) is enabled in the
    // primary context (idempotent; another runtime instance in the process may or may not have done it already)
    for (uint32_t g = 0; g < world; g++) {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, shard_ptrs[g]) == cudaSuccess && a.type == cudaMemoryTypeDevice && a.device != dev) {
            const cudaError_t e = cudaDeviceEnablePeerAccess(a.device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
                cudaFreeAsync(w.base, st);
                return int(e);
            }
        }
        cudaGetLastError();
    }
    const uint8_t** d_ptrs = reinterpret_cast<const uint8_t**>(w.first);
    cudaError_t ce = cudaMemcpyAsync(d_ptrs, shard_ptrs, sizeof(uint8_t*) * world, cudaMemcpyHostToDevice, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);  // shard_ptrs is the caller's (pageable) array
    if (ce != cudaSuccess) {
        cudaFreeAsync(w.base, st);
        return int(ce);
    }
    prep_gather_shards_kernel<<<cdiv(n, 256), 256, 0, st>>>(d_ptrs, world, block_size, n_blocks, file_len, d_dst, seg_shift, w.pieces, w.counts);
    count_launch();
    return copy_pieces(w, n, seg_shift, dev, st);
}

}  // extern "C"
