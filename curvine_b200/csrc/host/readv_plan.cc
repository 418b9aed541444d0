#include "readv_plan.h"

#include <algorithm>

namespace cv {

Err plan_shard(const FileBlocks& fb, int rank, int world, int64_t cap, std::vector<ShardJob>* out, int64_t* total) {
    out->clear();
    *total = 0;
    if (world <= 0 || rank < 0 || rank >= world) return Err::common("bad shard spec");
    const int64_t bs = fb.status.block_size;
    for (size_t b = static_cast<size_t>(rank), j = 0; b < fb.block_locs.size(); b += static_cast<size_t>(world), j++) {
        const int64_t blen = fb.block_locs[b].block.len;
        if (cap >= 0 && static_cast<int64_t>(j) * bs + blen > cap) return Err::common("destination too small for this shard");
        out->push_back(ShardJob{b, fb.starts[b], blen, static_cast<int64_t>(j) * bs});
        *total += blen;
    }
    return Err::ok();
}

// The rules only a scaled range has (check_cast, after its element alignment was checked): the scale geometry covers every element
// the range touches, without an int64 overflow anywhere.
static Err check_scale(const ReadvRange& r, int32_t i) {
    const ReadvScale& s = r.scale;
    const DtypeRow* sd = dtype_row(s.dtype);
    if (!sd || !sd->flt) return Err::common(str_printf("readv: range %d has an unknown scale dtype code %d", i, s.dtype));
    if (s.block_rows < 1 || s.block_cols < 1 || s.view_cols < 1 || s.rows < 1 || s.cols < 1)
        return Err::common(str_printf("readv: range %d: block_rows, block_cols, cols, scale_rows and scale_cols must be at least 1", i));
    if (s.first_elem < 0) return Err::common(str_printf("readv: range %d has a negative first_elem (%lld)", i, (long long)s.first_elem));
    const int64_t need = s.view_cols / s.block_cols + (s.view_cols % s.block_cols != 0);
    if (s.cols < need)
        return Err::common(str_printf("readv: range %d: scale_cols %lld < ceil(cols / block_cols) = %lld", i, (long long)s.cols, (long long)need));
    int64_t bytes;
    if (__builtin_mul_overflow(s.rows, s.cols, &bytes) || __builtin_mul_overflow(bytes, sd->size, &bytes))
        return Err::common(str_printf("readv: range %d: scale_rows * scale_cols * scale size overflows", i));
    if (r.rows == 0 || r.row_len == 0) return Err::ok();
    // the last view element the range touches: first_elem + (rows - 1) * file_pitch / src size + row_len / src size - 1
    const int64_t ss = dtype_size(r.src_dtype);
    int64_t last;
    if (__builtin_mul_overflow(r.rows - 1, r.rows > 1 ? r.file_pitch / ss : 0, &last) || __builtin_add_overflow(last, r.row_len / ss - 1, &last) ||
        __builtin_add_overflow(last, s.first_elem, &last))
        return Err::common(str_printf("readv: range %d: its last view element overflows int64", i));
    const int64_t srow = last / s.view_cols / s.block_rows;
    if (srow >= s.rows)
        return Err::common(str_printf("readv: range %d: view element %lld maps to scale row %lld, but the scale has %lld rows", i, (long long)last,
                                      (long long)srow, (long long)s.rows));
    return Err::ok();
}

// The rules only a converting range has (plan_readv)
static Err check_cast(const FileBlocks& fb, const ReadvRange& r, int32_t i) {
    for (int32_t dt : {r.src_dtype, r.dst_dtype})
        if (!dtype_row(dt)) return Err::common(str_printf("readv: range %d has an unknown dtype code %d", i, dt));
    if (r.scaled() && !is_f8(r.src_dtype))
        return Err::common(str_printf("readv: range %d is scaled but its source dtype %d is not F8_E4M3 or F8_E5M2", i, r.src_dtype));
    if (is_f8(r.dst_dtype) && (r.cast() || r.scaled()))
        return Err::common(str_printf("readv: range %d converts to F8 dtype %d: F8 is a source type only", i, r.dst_dtype));
    if (!r.cast()) return Err::ok();
    // F8 destinations are refused above: what is left here is CV_DTYPE_NONE on either side
    if (!(kDtypes[r.src_dtype].flt || is_f8(r.src_dtype)) || !kDtypes[r.dst_dtype].flt)
        return Err::common(str_printf("readv: range %d converts dtype %d to %d: conversions are between F32, F16 and BF16 only", i, r.src_dtype, r.dst_dtype));
    const int64_t ss = dtype_size(r.src_dtype), ds = dtype_size(r.dst_dtype);
    if (r.file_off % ss || r.row_len % ss || (r.rows > 1 && r.file_pitch % ss))
        return Err::common(str_printf("readv: range %d: file_off, row_len and file_pitch must be multiples of the source element size (%lld)", i, (long long)ss));
    if (reinterpret_cast<uintptr_t>(r.dst) % ds || (r.rows > 1 && r.dst_pitch % ds))
        return Err::common(str_printf("readv: range %d: the destination and dst_pitch must be multiples of the destination element size (%lld)", i, (long long)ds));
    if (fb.status.block_size % ss)
        return Err::common(str_printf("readv: range %d: the file's block size %lld is not a multiple of the source element size (%lld)", i,
                                      (long long)fb.status.block_size, (long long)ss));
    return r.scaled() ? check_scale(r, i) : Err::ok();
}

Err plan_readv(const FileBlocks& fb, const ReadvRange* ranges, int32_t n, std::vector<ReadvBlock>* blocks, std::vector<ReadvSpan>* spans) {
    blocks->clear(), spans->clear();
    if (n < 0) return Err::common(str_printf("readv: negative range count %d", n));
    if (n > 0 && !ranges) return Err::common("readv: null range table");
    const int64_t flen = fb.status.len;
    std::vector<int32_t> order;
    std::vector<int64_t> extent(static_cast<size_t>(n));  // file bytes from row 0's first byte to the last row's last byte
    for (int32_t i = 0; i < n; i++) {
        const ReadvRange& r = ranges[i];
        if (r.row_len < 0) return Err::common(str_printf("readv: range %d has a negative length (%lld)", i, (long long)r.row_len));
        if (r.rows < 0) return Err::common(str_printf("readv: range %d has a negative row count (%lld)", i, (long long)r.rows));
        if (r.file_pitch < 0 || r.dst_pitch < 0) return Err::common(str_printf("readv: range %d has a negative pitch", i));
        CV_RETURN_IF_ERR(check_cast(fb, r, i));
        const int64_t dst_row = dst_row_len(r);
        if (r.rows > 1 && (r.file_pitch < r.row_len || r.dst_pitch < dst_row))
            return Err::common(str_printf("readv: range %d has a pitch shorter than its row length (%lld)", i, (long long)r.row_len));
        int64_t& ext = extent[static_cast<size_t>(i)];
        ext = r.rows == 0 ? 0 : r.row_len;
        for (int64_t pitch : {r.file_pitch, r.dst_pitch})
            if (r.rows > 1 && pitch > 0 && r.rows - 1 > (INT64_MAX - std::max(r.row_len, dst_row)) / pitch)
                return Err::common(str_printf("readv: range %d: (rows - 1) * pitch + row_len overflows", i));
        if (r.rows > 1) ext += (r.rows - 1) * r.file_pitch;
        if (r.file_off < 0 || r.file_off > flen || ext > flen - r.file_off)
            return Err::common(str_printf("readv: range %d [%lld, +%lld) lies outside the file (%lld bytes)", i, (long long)r.file_off, (long long)ext, (long long)flen));
        if (r.row_len > 0 && r.rows > 0) order.push_back(i);
    }
    std::sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return ranges[a].file_off < ranges[b].file_off; });
    for (size_t k = 1; k < order.size(); k++)
        if (ranges[order[k]].file_off < ranges[order[k - 1]].file_off + extent[static_cast<size_t>(order[k - 1])])
            return Err::common(str_printf("readv: ranges %d and %d overlap in the file", order[k - 1], order[k]));
    for (int32_t i : order) {
        const ReadvRange& r = ranges[i];
        const int64_t L = r.row_len, R = r.rows, P = R > 1 ? r.file_pitch : L, off = r.file_off;
        // a converting range's in-row offsets scale to destination bytes; its row offsets are dst_pitch apart as for any range
        const int64_t ss = r.cast() ? dtype_size(r.src_dtype) : 1, ds = r.cast() ? dtype_size(r.dst_dtype) : 1;
        // next byte to place: column `col` of row `row`.  Every pass of the loop handles one touched block, in file order.
        int64_t row = 0, col = 0;
        while (row < R) {
            const int64_t q = off + row * P + col;
            int64_t boff;
            size_t idx;
            CV_RETURN_IF_ERR(fb.get_read_block(q, &boff, &idx));
            const int64_t bs = q - boff, be = bs + fb.block_locs[idx].block.len;
            if (blocks->empty() || blocks->back().block != idx) blocks->push_back(ReadvBlock{idx, false, spans->size(), 0});
            Err bad;
            auto emit = [&](int64_t at, int64_t len, int64_t rows, int64_t dst_off) {
                if (((at - off) | len) % ss)  // only a file whose blocks are not all block_size long gets here
                    bad = Err::common(str_printf("readv: range %d: an element straddles the edge of block %zu", i, idx));
                spans->push_back(ReadvSpan{at - bs, len, rows, dst_off, i});
                blocks->back().n_spans++;
            };
            // the row in progress, when it began in an earlier block or runs past this one: clipped by the block's edge
            if (col > 0 || off + row * P + L > be) {
                const int64_t take = std::min(L - col, be - q);
                emit(q, take, 1, row * r.dst_pitch + col / ss * ds);
                col += take;
                if (bad) return bad;
                if (col < L) continue;  // it goes on in the next block
                row++, col = 0;
            }
            // the whole rows that start and end inside the block
            if (row < R && off + row * P + L <= be) {
                const int64_t last = std::min(R - 1, (be - L - off) / P);
                emit(off + row * P, L, last - row + 1, row * r.dst_pitch);
                row = last + 1;
            }
            // a row that starts inside the block and runs past its end
            if (row < R && off + row * P < be) {
                const int64_t take = be - (off + row * P);
                emit(off + row * P, take, 1, row * r.dst_pitch);
                col = take;
            }
            if (bad) return bad;
            // otherwise the next row starts in a later block: the next pass looks that block up directly
        }
    }
    for (ReadvBlock& b : *blocks) {
        const ReadvSpan& s = (*spans)[b.first_span];
        b.direct = b.n_spans == 1 && s.rows == 1 && s.block_off == 0 && s.len == fb.block_locs[b.block].block.len && !ranges[s.range].cast();
    }
    return Err::ok();
}

}  // namespace cv
