/*
 * curvine_b200_kernels.h -- lower boundary: host -> CUDA (sm_90a) launchers.
 *
 * The "thin extern C layer" the north_star asks for (SURVEY.md §8b, lower boundary):
 * plain launchers, no C++ or torch types in signatures, the caller owns all memory,
 * everything is asynchronous on a caller-supplied stream, every entry point returns a
 * cudaError_t as int (0 == cudaSuccess) and never throws or aborts.  A Rust host binds
 * these with an `extern "C"` block 1:1 (see INTEGRATION.md).
 *
 * What each launcher replaces in the reference (paths relative to the CurvineIO/curvine source tree):
 *   cvk_crc_blocks      Utils::crc32 on the caller thread   orpc/src/common/utils.rs:73-75,
 *                       as used per read buffer by          curvine-tests/src/curvine_bench.rs:37-48,222-231
 *   cvk_unpack_frames   RpcFrame::receive + decode_protocol orpc/src/handler/rpc_frame.rs:222-264,
 *                       + RawClient::check_response         orpc/src/message/rpc_message.rs:326-338,
 *                       + Reader::read's copy_to_slice      orpc/src/client/raw_client.rs:100-116,
 *                                                           curvine-common/src/fs/reader.rs:71-81
 *   cvk_gather_pages    Reader::fuse_read + as_iovec/writev curvine-common/src/fs/reader.rs:101-124,
 *                                                           curvine-fuse/src/session/fuse_response.rs:49-60,171-175
 *   cvk_gather_strided  (no reference counterpart: the rows of tensor-parallel slices of a checkpoint, strided reads)
 *   cvk_gather_cast     (no reference counterpart: checkpoint tensors converted to another float type on load)
 *   cvk_gather_cast_scaled  (no reference counterpart: FP8 checkpoint weights dequantized with their scales on load)
 *   cvk_pack_frames     RpcMessage::encode_protocol +      orpc/src/message/rpc_message.rs:301-311,
 *                       RpcFrame::send/write_region          orpc/src/handler/rpc_frame.rs:97-121,205-220
 *                       (worker ReadHandler::read response)  curvine-server/src/worker/handler/read_handler.rs:143-183
 *   cvk_deinterleave_blocks, cvk_gather_shards_p2p  (no reference counterpart: model-distribution exchange, config C4)
 */
#ifndef CURVINE_B200_KERNELS_H
#define CURVINE_B200_KERNELS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* cv_stream_t; /* cudaStream_t */

/* Memory access rule of every launcher below.  Destinations are written exactly: no byte outside a destination range is touched.
 * Sources are read in whole 16-byte ALIGNED vectors: up to 15 bytes in front of and behind a source range may be read as well, never
 * outside the aligned 16-byte granules that hold the range -- so never across a page, a cudaMalloc granule (256 B) or a pinned-ring
 * slot.  (Checked by tools/sanitize_kernels.sh on the host-side SIMT shim and by compute-sanitizer memcheck on the device.) */

#define CV_POLY_IEEE 0       /* CRC-32/ISO-HDLC == crc32fast::hash == zlib.crc32 (reference tools) */
#define CV_POLY_CASTAGNOLI 1 /* CRC-32C (north_star's added integrity check) */

/* orpc wire constants (rpc_message.rs:26-41) */
#define CV_PROTOCOL_SIZE 22
#define CV_HEAD_SIZE 18
#define CV_MAX_DATA_SIZE (16 * 1024 * 1024)
#define CV_CODE_READ_BLOCK 81

/* frame validation error bits written to d_err_flags[frame] by cvk_unpack_frames */
#define CV_FERR_TOTAL_LEN 0x01u  /* total_len != 18 + header_len + data_len */
#define CV_FERR_HEADER_LEN 0x02u /* header_len differs from the descriptor */
#define CV_FERR_CODE 0x04u
#define CV_FERR_STATUS 0x08u     /* e.g. an error response (0x13) where data (0x03) was expected */
#define CV_FERR_REQ_ID 0x10u     /* raw_client.rs:100-116 echo check */
#define CV_FERR_SEQ_ID 0x20u
#define CV_FERR_DATA_RANGE 0x40u /* data_len < 0 or > 16 MiB (rpc_message.rs:329-334) */

/* One received frame: prefix at d_wire + wire_off, then header_len bytes, then data_len payload bytes. */
typedef struct CvFrameDesc {
    uint64_t wire_off;   /* offset of the 22-byte prefix inside the wire image */
    uint64_t dst_off;    /* destination offset of the payload inside d_dst */
    uint32_t data_len;   /* expected payload bytes */
    uint32_t header_len; /* expected protobuf header bytes (0 for Running data responses) */
    int64_t req_id;      /* expected echoes */
    int32_t seq_id;
    uint32_t block;      /* dense block index; frames of one block are contiguous and in stream order */
    uint8_t code;        /* expected code (81) */
    uint8_t status;      /* expected status byte (0x03 = Running|Success) */
    uint8_t pad_[2];
    uint32_t tail_clip;  /* K2: the last tail_clip payload bytes of the frame are validated as part of the frame but not copied
                          * (a ranged read whose last chunk runs past the wanted range); 0 for whole frames.  K4 ignores it. */
} CvFrameDesc;

/* A whole pipelined block response stream with closed-form frame offsets:
 * frame f starts at wire_off + f*(22+chunk_size), carries min(chunk_size, block_len - f*chunk_size) bytes,
 * seq_id = first_seq_id + f.  Expanded on the device into CvFrameDesc by cvk_expand_streams. */
typedef struct CvStreamDesc {
    uint64_t wire_off;
    uint64_t dst_off;
    uint64_t block_len;
    int64_t req_id;
    uint32_t chunk_size;
    int32_t first_seq_id;
    uint32_t block;
    uint32_t first_frame; /* index of this stream's first frame in the expanded descriptor table */
    uint8_t code;
    uint8_t status;
    uint8_t pad_[2];
    uint32_t tail_clip;   /* bytes at the end of the stream (inside its last frame) that are received but not delivered */
} CvStreamDesc;

/* scatter/gather segment: d_dst[dst_off .. dst_off+len) = d_src[src_off .. src_off+len) */
typedef struct CvSeg {
    uint64_t src_off;
    uint64_t dst_off;
    uint64_t len;
} CvSeg;

/* strided segment: rows equally spaced copies of len bytes,
 * d_dst[dst_off + k*dst_pitch .. +len) = d_src[src_off + k*src_pitch .. +len) for k < rows */
typedef struct CvStridedSeg {
    uint64_t src_off;
    uint64_t dst_off;
    uint64_t len;
    uint64_t rows;
    uint64_t src_pitch;
    uint64_t dst_pitch;
} CvStridedSeg;

/* element types of cvk_gather_cast and of cast reads (CvCastRange).  CV_DTYPE_NONE: bytes as stored, no conversion.  The two FP8
 * codes are source types only, converted by cvk_gather_cast_scaled: E4M3 is torch's float8_e4m3fn (no infinities, 0x7f / 0xff are
 * NaN), E5M2 is float8_e5m2. */
#define CV_DTYPE_NONE 0
#define CV_DTYPE_F32 1
#define CV_DTYPE_F16 2
#define CV_DTYPE_BF16 3
#define CV_DTYPE_F8_E4M3 4
#define CV_DTYPE_F8_E5M2 5

/* Work chunks of one row of `elems` elements in cvk_gather_cast: a chunk is 8 elements whose destination starts 16-byte aligned, plus
 * a head chunk for the elements in front of the first aligned one. */
#define CV_CAST_ROW_CHUNKS(elems) ((elems) ? ((uint64_t)(elems) + 14) / 8 : 0)

/* cast segment: rows equally spaced rows of elems elements, converted from src_dtype to dst_dtype,
 * d_dst[dst_off + k*dst_pitch ..) = convert(d_src[src_off + k*src_pitch ..)) for k < rows (offsets and pitches in bytes).
 * `first` is the work distribution, filled by the host: the exclusive prefix over the table of rows * CV_CAST_ROW_CHUNKS(elems). */
typedef struct CvCastSeg {
    uint64_t src_off;
    uint64_t dst_off;
    uint64_t elems;      /* elements per row */
    uint64_t rows;
    uint64_t src_pitch;
    uint64_t dst_pitch;
    uint64_t first;      /* first work chunk of this segment */
    int32_t src_dtype;   /* CV_DTYPE_F32 / _F16 / _BF16 */
    int32_t dst_dtype;
} CvCastSeg;             /* 64 bytes */

/* scale of a cast segment in cvk_gather_cast_scaled (one per CvCastSeg, same index).  The segment's elements are elements of a
 * weight seen as a row-major 2-D view [V_rows, cols]: element e of segment row k is view element view0 + k*view_step + e, and view
 * element (i, j) is multiplied by scale[(i / block_rows) * scale_cols + j / block_cols] before it is rounded to the destination.
 * scale == NULL: the segment is not scaled. */
typedef struct CvScaleSeg {
    const void* scale;   /* scale elements in HBM, row-major */
    uint64_t block_rows; /* view rows per scale row */
    uint64_t block_cols; /* view columns per scale column */
    uint64_t scale_cols;
    uint64_t cols;       /* view columns */
    uint64_t view0;      /* view element of the segment's row 0, element 0 */
    uint64_t view_step;  /* view elements between the starts of two segment rows */
    int32_t scale_dtype; /* CV_DTYPE_F32 / _F16 / _BF16 */
    int32_t pad;
} CvScaleSeg;            /* 64 bytes */

/* Build the per-device constant tables (both polynomials).  Optional: every launcher does it lazily. */
int cvk_init(int device);

/* K1: d_crc_out[i] = CRC(d_base[d_off[i] .. d_off[i]+d_len[i])) for i < n.  Any alignment, any length
 * (0 -> 0).  total_bytes = sum of d_len (an upper bound is fine; sizes the scratch space).
 * Algorithmic bytes: reads N, writes 4 per block. */
int cvk_crc_blocks(const uint8_t* d_base, const uint64_t* d_off, const uint64_t* d_len, uint32_t n, int poly,
                   uint64_t total_bytes, uint32_t* d_crc_out, cv_stream_t stream);

/* d_n_bad += #{i : d_crc[i] != d_expect[i]} ; d_bad_mask[i] = mismatch (optional, may be NULL). */
int cvk_verify_crcs(const uint32_t* d_crc, const uint32_t* d_expect, uint32_t n, uint32_t* d_n_bad,
                    uint8_t* d_bad_mask, cv_stream_t stream);

/* Same, but entries with d_skip[i] != 0 are not compared (blocks the manifest holds no CRC for, holes, partial
 * ranges): one such block no longer switches the comparison off for its neighbours.  d_skip may be NULL. */
int cvk_verify_crcs_masked(const uint32_t* d_crc, const uint32_t* d_expect, const uint8_t* d_skip, uint32_t n,
                           uint32_t* d_n_bad, uint8_t* d_bad_mask, cv_stream_t stream);

/* K2: validate n frame prefixes, gather payloads to d_dst and CRC them in the same pass.
 * d_block_crc[b] (b < n_blocks) = CRC of block b's payload bytes in frame order; d_err_flags[f] = CV_FERR_*.
 * Either output may be NULL.  Algorithmic bytes: reads N + 22F, writes N. */
int cvk_unpack_frames(const uint8_t* d_wire, const CvFrameDesc* d_desc, uint32_t n_frames, uint32_t n_blocks,
                      uint8_t* d_dst, int poly, uint64_t total_bytes, uint32_t* d_block_crc,
                      uint32_t* d_err_flags, cv_stream_t stream);

/* Expand n_streams regular block streams into n_frames CvFrameDesc entries (device side). */
int cvk_expand_streams(const CvStreamDesc* d_streams, uint32_t n_streams, CvFrameDesc* d_desc_out,
                       uint32_t n_frames, cv_stream_t stream);

/* K3: page scatter/gather, arbitrary alignment.  Algorithmic bytes: reads N, writes N. */
int cvk_gather_pages(const uint8_t* d_src, const CvSeg* d_segs, uint32_t n, uint64_t total_bytes, uint8_t* d_dst,
                     cv_stream_t stream);

/* K3 over 2D descriptors: every row of every segment, arbitrary alignment (rows of different segments must not overlap in d_dst).
 * The rows are expanded into walker pieces on the device, in trains of at most 2^22 rows (cvk_tune(6, ...)), so the workspace
 * does not grow with the row count.  Sizing the trains needs the row total: the launcher reads the n descriptors back, so it
 * returns once the work queued on `stream` before it has finished (the copy itself stays asynchronous).
 * total_bytes = sum of len * rows.  Algorithmic bytes: reads N, writes N. */
int cvk_gather_strided(const uint8_t* d_src, const CvStridedSeg* d_segs, uint32_t n, uint64_t total_bytes, uint8_t* d_dst,
                       cv_stream_t stream);

/* K5: gather with a dtype conversion, every row of every segment: F32, F16 and BF16 into one another, IEEE round-to-nearest-even
 * (subnormals, signed zeros, infinities; F32 -> F16 overflows to inf), bit-identical to torch's CPU Tensor.to() for every non-NaN input;
 * a NaN stays a NaN (its payload may differ).  F16 <-> BF16 goes through F32, which is exact: one rounding.  A segment with
 * src_dtype == dst_dtype is a copy; one with a code other than the three is skipped.  Sources and destinations need only their
 * element alignment; a row is converted in chunks of 8 elements whose destination is 16-byte aligned (a scalar head and tail around
 * them), the chunks of all segments spread over all SMs, and the launcher neither reads the table back nor synchronises.
 * total_elems = sum of elems * rows (sizes the grid; 0 launches nothing).  Rows of different segments must not overlap in d_dst.
 * Algorithmic bytes: reads N * src size, writes N * dst size. */
int cvk_gather_cast(const uint8_t* d_src, const CvCastSeg* d_segs, uint32_t n, uint64_t total_elems, uint8_t* d_dst, cv_stream_t stream);

/* K5, scaled instance: cvk_gather_cast with FP8 sources (CV_DTYPE_F8_E4M3 / _E5M2, decoded exactly) and a scale per element.
 * d_scales[i] belongs to d_segs[i].  A segment with a scale gives y = round_dst(f32(x) * f32(s)): one IEEE F32 multiply (never
 * contracted, denormals kept), rounded once to dst_dtype as in cvk_gather_cast -- bit-identical to torch's CPU
 * (x.float() * s.float()).to(dst) for every non-NaN result.  A segment without one converts as cvk_gather_cast does (FP8 exactly).
 * The scale of an element is found from its view position once per 8-element chunk and stepped from there; the scale element index
 * must lie inside the caller's scale buffer (cv_readv_scaled_device validates it).  FP8 sources need no alignment; whole chunks read
 * them in one 8-byte load when it is aligned.  d_scales may be NULL only when n == 0.  Algorithmic bytes: reads N * src size plus
 * the scales, writes N * dst size. */
int cvk_gather_cast_scaled(const uint8_t* d_src, const CvCastSeg* d_segs, const CvScaleSeg* d_scales, uint32_t n, uint64_t total_elems,
                           uint8_t* d_dst, cv_stream_t stream);

/* K4: worker-side inverse of K2.  For frame f: write the 22-byte prefix (+ no header) at
 * d_wire + d_desc[f].wire_off, copy d_src[dst_off .. +data_len) behind it, and CRC the source bytes
 * (d_block_crc as in K2; may be NULL).  Algorithmic bytes: reads N, writes N + 22F. */
int cvk_pack_frames(const uint8_t* d_src, const CvFrameDesc* d_desc, uint32_t n_frames, uint32_t n_blocks,
                    uint8_t* d_wire, int poly, uint64_t total_bytes, uint32_t* d_block_crc, cv_stream_t stream);

/* After an all-gather of G rank shards, each holding its round-robin blocks back to back
 * (shard g slot j = file block j*G+g; slots are block_size bytes, shard stride shard_stride bytes),
 * restore file order: d_dst[b*block_size ..) = block b, for b < n_blocks; the last block may be short
 * (file_len).  Algorithmic bytes: reads N, writes N. */
int cvk_deinterleave_blocks(const uint8_t* d_gathered, uint64_t shard_stride, uint32_t world, uint64_t block_size,
                            uint64_t n_blocks, uint64_t file_len, uint8_t* d_dst, cv_stream_t stream);

/* Fused all-gather + de-interleave over peer memory (config C4, NVLink/NVSwitch): shard_ptrs[g] (HOST array of
 * `world` device pointers, the local shard and the peers' shards mapped with CUDA IPC / peer access) is rank g's shard
 * in the layout cv_read_device_sharded produces; every block is pulled straight from its owner's HBM into file order
 * at d_dst -- no intermediate gathered buffer, no second pass.  Algorithmic bytes: reads N (N*(G-1)/G of it over
 * NVLink), writes N. */
int cvk_gather_shards_p2p(const uint8_t* const* shard_ptrs, uint32_t world, uint64_t block_size, uint64_t n_blocks,
                          uint64_t file_len, uint8_t* d_dst, cv_stream_t stream);

/* Time the dominant row-walker kernel (K1/K2/K4 bodies) with CUDA events on the launching stream.
 * enable(1) starts collecting (and clears), collect() synchronises the recorded events and returns the summed
 * duration in ms and the number of walker launches; enable(0) stops. */
int cvk_profile_enable(int on);
int cvk_profile_collect(double* walk_ms_total, uint32_t* walk_launches);

/* Tuning hook: forces the other side of launch choices the library otherwise makes from the input.  what 4: segment size
 * 2^value bytes (12..20) for every launcher instead of the size-derived choice, 0 = back to automatic; what 5: 0 routes inputs
 * of at most ~1 MiB through the general launch train instead of the single-launch small-input kernels (default 1); what 6: rows
 * per train of cvk_gather_strided, 1..2^22, 0 = back to the default 2^22.  Any other what, or a value out of range, returns
 * cudaErrorInvalidValue.  Process-wide; results are identical for every setting. */
int cvk_tune(int what, int value);

/* Number of kernel launches issued by this library in this process (bench.py's gpu_launches claim). */
uint64_t cvk_launch_count(void);

/* ---- cvh_*: the host-side CUDA plumbing a caller needs around the launchers above, so that a host written in a language without CUDA
 * bindings (the reference's Rust client with its own fetch loop: a `UnifiedReader::Cuda` that keeps RpcFrame::receive and hands the bytes
 * to K2) links nothing but this library.  Thin wrappers over the runtime; all return cudaError_t as int.
 *   cvh_pinned_alloc / cvh_pinned_free   page-locked host buffers: where received frames / pread chunks land so that the H2D copy is a DMA
 *                                        (replaces the BytesMut carved by FrameBuf::take_exact, orpc/src/handler/frame_buf.rs:58-70)
 *   cvh_host_register / _unregister      the same for memory the caller already owns (short-circuit: an mmap of the block file)
 *   cvh_device_alloc / cvh_device_free   device buffers (wire staging, destinations) for callers that have no allocator of their own
 *   cvh_h2d_async                        dst[0..n) <- pinned src on copy_stream; done_event (may be NULL) is recorded behind the copy
 *   cvh_d2h_async                        the way back for results (per-block CRCs, error flags)
 *   cvh_stream_* / cvh_event_*           creation, ordering (stream waits for event) and completion of the two handle kinds the calls take */
typedef void* cv_event_t; /* cudaEvent_t */
int cvh_pinned_alloc(size_t bytes, void** out);
int cvh_pinned_free(void* p);
int cvh_host_register(void* p, size_t bytes);   /* page-lock memory the caller already owns (an mmap'ed block file, a receive buffer): cudaHostRegister */
int cvh_host_unregister(void* p);
int cvh_device_alloc(size_t bytes, void** out);
int cvh_device_free(void* d_p);
int cvh_h2d_async(void* d_dst, const void* h_src, size_t n, cv_stream_t copy_stream, cv_event_t done_event);
int cvh_d2h_async(void* h_dst, const void* d_src, size_t n, cv_stream_t stream, cv_event_t done_event);
int cvh_stream_create(cv_stream_t* out);  /* non-blocking stream on the current device */
int cvh_stream_destroy(cv_stream_t s);
int cvh_stream_synchronize(cv_stream_t s);
int cvh_stream_wait_event(cv_stream_t s, cv_event_t e);
int cvh_event_create(cv_event_t* out);    /* timing disabled */
int cvh_event_destroy(cv_event_t e);
int cvh_event_record(cv_event_t e, cv_stream_t s);
int cvh_event_synchronize(cv_event_t e);
int cvh_event_query(cv_event_t e);        /* 0 = complete, cudaErrorNotReady (600) = still pending */

#ifdef __cplusplus
}
#endif
#endif
