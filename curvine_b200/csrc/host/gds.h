// GPUDirect Storage for the SSD/HDD tiers (SURVEY.md 8f-2): cuFileRead straight into the destination in HBM, no pinned host
// ring in between.  libcufile is dlopen'ed at first use (the product library carries no link-time dependency on it); when it is
// missing, when the driver cannot be opened, or when a file cannot be registered, the caller falls back to the pinned ring and
// says so in the read stats.  Without the nvidia-fs kernel module GDS is reported unavailable and cuFile is never opened: it could
// only run its compatibility mode (POSIX reads into its own bounce buffers + copies), whose driver open can block indefinitely.
#pragma once
#include "common.h"

namespace cv {

struct GdsInfo {
    bool available = false;  // nvidia-fs loaded, libcufile loaded and cuFileDriverOpen succeeded
    std::string detail;
};

const GdsInfo& gds_info();  // probes once per process
// n bytes of `path` starting at file_off -> d_dst (device memory of the current device).  kUnsupported when GDS cannot serve it.
Err gds_read(const std::string& path, void* d_dst, int64_t n, int64_t file_off);
std::string gds_last_refusal();  // why the first file that was turned away was turned away ("" if none was)
void gds_forget(const std::string& path);  // drop the cached handle (file replaced / context teardown: "" = all)

}  // namespace cv
