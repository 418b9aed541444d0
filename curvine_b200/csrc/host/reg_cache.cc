#include "reg_cache.h"

namespace cv {

// (inode, size, mtime_ns) of a block file: what a cached mapping of it is revalidated by
static void file_stamp(const struct stat& st, std::vector<uint64_t>* stamps) {
    stamps->push_back(static_cast<uint64_t>(st.st_ino)), stamps->push_back(static_cast<uint64_t>(st.st_size));
    stamps->push_back(static_cast<uint64_t>(st.st_mtim.tv_sec) * 1000000000ull + static_cast<uint64_t>(st.st_mtim.tv_nsec));
}

Err map_and_register(const std::vector<std::string>& paths, const std::vector<int64_t>& lens, std::shared_ptr<RegMapping>* out,
                     std::vector<uint64_t>* stamps_out) {
    size_t total = 0;
    for (size_t i = 0; i < paths.size(); i++) {
        if (i + 1 < paths.size() && lens[i] % 4096) return Err::common("block length is not page aligned");
        total += page_up(static_cast<size_t>(lens[i]));
    }
    std::shared_ptr<RegMapping> m(new RegMapping());
    void* base = mmap(nullptr, total, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (base == MAP_FAILED) return Err::io(str_printf("mmap reserve: %s", strerror(errno)));
    m->base = static_cast<uint8_t*>(base), m->bytes = total;
    size_t off = 0;
    for (size_t i = 0; i < paths.size(); i++) {
        // cudaHostRegister needs a writable shared mapping here (cudaHostRegisterReadOnly is not supported on this
        // platform); nothing ever writes through it.  Read-only block files fall back to the pinned ring.
        const int fd = ::open(paths[i].c_str(), O_RDWR | O_CLOEXEC);
        if (fd < 0) return Err(kUnsupported, str_printf("open %s read-write: %s", paths[i].c_str(), strerror(errno)));
        struct stat st;
        fstat(fd, &st);
        if (st.st_size < lens[i]) {
            ::close(fd);
            return Err::io("block file shorter than the block length");
        }
        file_stamp(st, &m->stamps);
        const size_t span = page_up(static_cast<size_t>(lens[i]));
        void* p = mmap(m->base + off, span, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_FIXED | MAP_POPULATE, fd, 0);
        ::close(fd);
        if (p == MAP_FAILED) return Err::io(str_printf("mmap %s: %s", paths[i].c_str(), strerror(errno)));
        off += span;
    }
    cudaError_t e = cudaHostRegister(m->base, total, cudaHostRegisterDefault);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return Err(kUnsupported, str_printf("cudaHostRegister(%zu): %s", total, cudaGetErrorString(e)));
    }
    m->registered = true;
    *stamps_out = m->stamps;
    *out = std::move(m);
    return Err::ok();
}

bool stat_stamps(const std::vector<std::string>& paths, std::vector<uint64_t>* stamps) {
    stamps->clear();
    for (const auto& p : paths) {
        struct stat st;
        if (stat(p.c_str(), &st) != 0) return false;
        file_stamp(st, stamps);
    }
    return true;
}

}  // namespace cv
