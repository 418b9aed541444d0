// Read planners: which blocks of a file a sharded or vectored device read touches, and where each span of them goes.  Geometry and
// validation over a FileBlocks only: no CUDA here, so the plans build, run and are tested without a GPU (cv_shard_plan, cv_readv_*_plan).
#pragma once
#include <iterator>
#include <vector>

#include "../../../include/curvine_b200_kernels.h"
#include "client.h"

namespace cv {

// The element types of cast reads, one row per CV_DTYPE_* code (the row's index).  kernels.cu keeps its own device-side sizes.
struct DtypeRow {
    int64_t size;  // bytes per element; CV_DTYPE_NONE: bytes as stored
    bool f8;       // F8_E4M3, F8_E5M2: a source type only
    bool flt;      // F32, F16, BF16: a conversion target and a scale dtype
};
inline constexpr DtypeRow kDtypes[] = {
    {1, false, false},  // CV_DTYPE_NONE
    {4, false, true},   // CV_DTYPE_F32
    {2, false, true},   // CV_DTYPE_F16
    {2, false, true},   // CV_DTYPE_BF16
    {1, true, false},   // CV_DTYPE_F8_E4M3
    {1, true, false},   // CV_DTYPE_F8_E5M2
};
static_assert(std::size(kDtypes) == CV_DTYPE_F8_E5M2 + 1, "one row per CV_DTYPE_* code");

// The row of code `dt`; nullptr for a code outside the table.
inline const DtypeRow* dtype_row(int32_t dt) { return dt >= 0 && dt < static_cast<int32_t>(std::size(kDtypes)) ? &kDtypes[dt] : nullptr; }
// These take a code the planner accepted (check_cast, check_scale).
inline int64_t dtype_size(int32_t dt) { return kDtypes[dt].size; }
inline bool is_f8(int32_t dt) { return kDtypes[dt].f8; }

// Round-robin shard of a file: block b -> rank b % world (the analogue of slice_id % read_parallel,
// fs_reader_parallel.rs:112-122).  Slot j of the rank's destination (block_size bytes each) holds block j*world+rank.
struct ShardJob {
    size_t block;      // index into FileBlocks::block_locs
    int64_t file_off;  // where the block starts in the file
    int64_t len;
    int64_t dst_off;   // j * block_size
};
Err plan_shard(const FileBlocks& fb, int rank, int world, int64_t cap, std::vector<ShardJob>* out, int64_t* total);

// Vectored read: n strided ranges of one file -> n destinations.  A range is `rows` rows of `row_len` bytes: row k is file bytes
// [file_off + k*file_pitch, +row_len) and lands at dst + k*dst_pitch (a plain byte range is one row).  The plan lists every block a range
// touches, in file order, with the spans of it that go to which range.  A block is direct when one span of one row covers all of it: it
// lands in place as an ordinary whole-block job.  Every other touched block is a boundary block: it is fetched whole into device staging,
// verified there like any whole block, and its spans are delivered from the staging by K3.  A range whose src_dtype differs from its
// dst_dtype converts its elements (CV_DTYPE_*): its file side is in source bytes, its destination side (dst, dst_pitch, a span's dst_off)
// in destination bytes, and none of the blocks it touches is direct, so each is verified before K5 converts it out of the staging.
// A scaled range (scale.ptr != nullptr, FP8 sources only) also multiplies every element by its scale (CvScaledRange).
struct ReadvScale {
    const void* ptr = nullptr;
    int32_t dtype = CV_DTYPE_NONE;
    int64_t rows = 0, cols = 0, block_rows = 0, block_cols = 0, view_cols = 0, first_elem = 0;
};
struct ReadvRange {
    int64_t file_off, row_len;
    uint8_t* dst;
    int64_t rows = 1, file_pitch = 0, dst_pitch = 0;  // the pitches only matter when rows > 1
    int32_t src_dtype = CV_DTYPE_NONE, dst_dtype = CV_DTYPE_NONE;
    ReadvScale scale;
    bool cast() const { return src_dtype != dst_dtype; }
    bool scaled() const { return scale.ptr != nullptr; }
};
struct ReadvSpan {
    int64_t block_off, len;  // row k < rows of the span: bytes [block_off + k*file_pitch, +len) of the block
    int64_t rows;
    int64_t dst_off;         // row k goes to ranges[range].dst + dst_off + k*dst_pitch (destination bytes)
    int32_t range;
};
struct ReadvBlock {
    size_t block;  // index into FileBlocks::block_locs
    bool direct;
    size_t first_span, n_spans;
};
// Ranges may come in any order.  An error: a negative row_len, rows or pitch; rows > 1 with a pitch shorter than row_len; an extent
// [file_off, file_off + (rows-1)*file_pitch + row_len) outside the file (or one that overflows); two ranges whose extents overlap in the
// file -- interleaved strided ranges included.  For one range and one block the rows that meet the block form at most three spans (a
// clipped first row, the whole rows, a clipped last row), computed without visiting the rows: O(ranges + touched blocks).  A converting
// range is an error besides when a dtype code is unknown, when it converts to or from CV_DTYPE_NONE, when an element could straddle two
// blocks or a source or destination element is misaligned (see cv_readv_cast_device), or when its dst_pitch is shorter than its
// destination row.  A scaled range is an error besides for the rules of cv_readv_scaled_device (all but the device-memory check).
Err plan_readv(const FileBlocks& fb, const ReadvRange* ranges, int32_t n, std::vector<ReadvBlock>* blocks, std::vector<ReadvSpan>* spans);

// A range's destination row in bytes: row_len converted to the destination element size.
inline int64_t dst_row_len(const ReadvRange& r) { return r.cast() ? r.row_len / dtype_size(r.src_dtype) * dtype_size(r.dst_dtype) : r.row_len; }

}  // namespace cv
