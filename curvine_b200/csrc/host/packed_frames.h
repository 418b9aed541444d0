// Running frames packed on the GPU (K4, cvk_pack_frames): the worker's HBM tier answers remote reads with them, the device writer
// sends them as write requests.  One module owns the frame descriptors and K4's buffer layout for both.
#pragma once
#include "../../../include/curvine_b200_kernels.h"
#include "common.h"

namespace cv {

// A packed stream of Running frames: frame f = wire + f*(22+chunk), carries min(chunk, remaining) bytes.  off0, total, chunk, req_id
// and first_seq describe the block read the HBM tier serves from it; the device writer only sends the image.
struct PackedStream {
    uint8_t* wire = nullptr;  // pinned host memory
    size_t wire_cap = 0;
    int64_t off0 = 0, total = 0, chunk = 0;
    int64_t req_id = 0;
    int32_t first_seq = 1;
    uint32_t crc32c = 0;  // CRC-32C of the packed payload, computed at the source by K4
    ~PackedStream();
};

// K4 over n bytes at d_src: Running frames of `chunk` payload bytes (code, status, req_id, seq ids first_seq..), packed into
// out->wire (grown as needed, pinned), their CRC-32C into out->crc32c and, when crc32 != nullptr, the CRC-32 of the same bytes (K1).
// Enqueued on `stream` and synchronised before it returns; the device buffer is released on every path.  n == 0 does nothing.
// The stream is a cv_stream_t so that the worker side, which holds a PackedStream, includes no CUDA header.
Err pack_running_frames(const uint8_t* d_src, int64_t n, int64_t chunk, uint8_t code, uint8_t status, int64_t req_id, int32_t first_seq,
                        cv_stream_t stream, PackedStream* out, uint32_t* crc32 = nullptr);

}  // namespace cv
