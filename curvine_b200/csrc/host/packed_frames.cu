#include "packed_frames.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

#include "wire.h"

namespace cv {

PackedStream::~PackedStream() {
    if (wire) cudaFreeHost(wire);
}

Err pack_running_frames(const uint8_t* d_src, int64_t n, int64_t chunk, uint8_t code, uint8_t status, int64_t req_id, int32_t first_seq,
                        cv_stream_t stream, PackedStream* out, uint32_t* crc32) {
    if (n == 0) return Err::ok();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const uint32_t nf = static_cast<uint32_t>((n + chunk - 1) / chunk);
    const size_t wire_bytes = static_cast<size_t>(n) + size_t(nf) * kProtocolSize;
    if (wire_bytes > out->wire_cap) {
        if (out->wire) cudaFreeHost(out->wire);
        out->wire = nullptr, out->wire_cap = 0;
        CU_TRY(cudaHostAlloc(&out->wire, wire_bytes, cudaHostAllocDefault));
        out->wire_cap = wire_bytes;
    }
    std::vector<CvFrameDesc> descs(nf);  // value-initialised: block, header_len, tail_clip and padding are 0
    for (uint32_t f = 0; f < nf; f++) {
        CvFrameDesc& d = descs[f];
        d.wire_off = uint64_t(f) * (kProtocolSize + chunk);
        d.dst_off = uint64_t(f) * chunk;  // offset of this chunk inside the source range
        d.data_len = static_cast<uint32_t>(std::min<int64_t>(chunk, n - int64_t(f) * chunk));
        d.req_id = req_id, d.seq_id = first_seq + static_cast<int32_t>(f), d.code = code, d.status = status;
    }
    // one device buffer: [wire image][descs][crc32c][off, len][crc32]; K1's table and result only when the CRC-32 is asked for
    const size_t o_desc = (wire_bytes + 255) & ~size_t(255), o_crc = o_desc + sizeof(CvFrameDesc) * nf, o_tab = (o_crc + 4 + 255) & ~size_t(255);
    const uint64_t tab[2] = {0, static_cast<uint64_t>(n)};
    uint8_t* d_buf = nullptr;
    CU_TRY(cudaMallocAsync(&d_buf, (crc32 ? o_tab : o_crc) + 64, st));
    Err e = [&]() -> Err {
        CU_TRY(cudaMemcpyAsync(d_buf + o_desc, descs.data(), sizeof(CvFrameDesc) * nf, cudaMemcpyHostToDevice, st));
        if (crc32) CU_TRY(cudaMemcpyAsync(d_buf + o_tab, tab, sizeof(tab), cudaMemcpyHostToDevice, st));
        CVK_TRY(cvk_pack_frames(d_src, reinterpret_cast<const CvFrameDesc*>(d_buf + o_desc), nf, 1, d_buf, CV_POLY_CASTAGNOLI, static_cast<uint64_t>(n),
                                reinterpret_cast<uint32_t*>(d_buf + o_crc), stream));
        if (crc32)
            CVK_TRY(cvk_crc_blocks(d_src, reinterpret_cast<const uint64_t*>(d_buf + o_tab), reinterpret_cast<const uint64_t*>(d_buf + o_tab + 8), 1,
                                   CV_POLY_IEEE, static_cast<uint64_t>(n), reinterpret_cast<uint32_t*>(d_buf + o_tab + 16), stream));
        CU_TRY(cudaMemcpyAsync(out->wire, d_buf, wire_bytes, cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaMemcpyAsync(&out->crc32c, d_buf + o_crc, 4, cudaMemcpyDeviceToHost, st));
        if (crc32) CU_TRY(cudaMemcpyAsync(crc32, d_buf + o_tab + 16, 4, cudaMemcpyDeviceToHost, st));
        return Err::ok();
    }();
    // freed and drained whatever failed: nothing this call enqueued outlives it
    const cudaError_t fe = cudaFreeAsync(d_buf, st);
    const cudaError_t se = cudaStreamSynchronize(st);
    if (!e && fe != cudaSuccess) e = Err::io(str_printf("cudaFreeAsync: %s", cudaGetErrorString(fe)));
    if (!e && se != cudaSuccess) e = Err::io(str_printf("cudaStreamSynchronize: %s", cudaGetErrorString(se)));
    return e;
}

}  // namespace cv
