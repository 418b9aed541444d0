// Shared host-side vocabulary: error kinds, result type, byte-order helpers.
#pragma once
#include <stdint.h>
#include <string.h>

#include <string>
#include <utility>

namespace cv {

// curvine-common/src/error/fs_error.rs:35-66 (ErrorKind); FFI return value is -(kind) (fs_error.rs:324-326).
enum ErrorKind : int32_t {
    kOk = 0,
    kIO = 1,
    kNotLeaderMaster = 2,
    kRaft = 3,
    kTimeout = 4,
    kPBDecode = 5,
    kPBEncode = 6,
    kFileAlreadyExists = 7,
    kFileNotFound = 8,
    kInvalidFileSize = 9,
    kParentNotDir = 10,
    kDirNotEmpty = 11,
    kAbnormalData = 12,
    kBlockIsWriting = 13,
    kBlockInfo = 14,
    kLease = 15,
    kInvalidPath = 16,
    kDiskOutOfSpace = 17,
    kInProgress = 18,
    kUnsupported = 19,
    kUfs = 20,
    kExpired = 21,
    kUnsupportedUfsRead = 22,
    kJobNotFound = 23,
    kPipeline = 24,
    kMinReplicasNotMet = 25,
    kCommon = 10000,
};

struct Err {
    int32_t kind = kOk;
    std::string msg;
    Err() = default;
    Err(int32_t k, std::string m) : kind(k), msg(std::move(m)) {}
    explicit operator bool() const { return kind != kOk; }  // true == failure
    static Err ok() { return Err(); }
    static Err common(std::string m) { return Err(kCommon, std::move(m)); }
    static Err io(std::string m) { return Err(kIO, std::move(m)); }
    Err ctx(const std::string& c) const { return Err(kind, c + ": " + msg); }
    int64_t libc_kind() const { return -static_cast<int64_t>(kind); }
};

#define CV_RETURN_IF_ERR(expr)      \
    do {                            \
        ::cv::Err e__ = (expr);     \
        if (e__) return e__;        \
    } while (0)

// A failed CUDA runtime call (CU_TRY) or cvk_* launcher (CVK_TRY) returns Err::io naming the call.  They name no CUDA type until they
// expand, so CUDA-free modules can include this header.
#define CU_TRY(x)                                                                                              \
    do {                                                                                                       \
        cudaError_t e_ = (x);                                                                                  \
        if (e_ != cudaSuccess) return ::cv::Err::io(::cv::str_printf("%s: %s", #x, cudaGetErrorString(e_)));  \
    } while (0)
#define CVK_TRY(x)                                                                                             \
    do {                                                                                                       \
        int e_ = (x);                                                                                          \
        if (e_ != 0) return ::cv::Err::io(::cv::str_printf("%s: %s", #x, cudaGetErrorString(cudaError_t(e_)))); \
    } while (0)

inline void put_be32(uint8_t* p, uint32_t v) { p[0] = v >> 24, p[1] = v >> 16, p[2] = v >> 8, p[3] = v; }
inline void put_be64(uint8_t* p, uint64_t v) {
    put_be32(p, static_cast<uint32_t>(v >> 32));
    put_be32(p + 4, static_cast<uint32_t>(v));
}
inline uint32_t get_be32(const uint8_t* p) {
    return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | uint32_t(p[3]);
}
inline uint64_t get_be64(const uint8_t* p) { return (uint64_t(get_be32(p)) << 32) | get_be32(p + 4); }

std::string str_printf(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
double now_sec();

}  // namespace cv
