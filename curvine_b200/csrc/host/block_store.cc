#include "block_store.h"

#include <dirent.h>
#include <errno.h>
#include <fcntl.h>
#include <stdlib.h>
#include <sys/stat.h>
#include <unistd.h>

#include "conf.h"
#include "numa.h"

namespace cv {

Err create_block_id(int64_t inode_id, int64_t seq, int64_t* out) {
    if (inode_id > kInodeIdMask) return Err::common(str_printf("inode id exceeds maximum value %lld", (long long)kInodeIdMask));
    if (seq > kSeqMask) return Err::common(str_printf("seq id exceeds maximum value %lld", (long long)kSeqMask));
    *out = ((inode_id & kInodeIdMask) << 24) | (seq & kSeqMask);
    return Err::ok();
}

std::string block_dir(const std::string& base, int64_t id) {
    const uint64_t u = static_cast<uint64_t>(id);
    return str_printf("%s/active/b%llu/b%llu", base.c_str(), (unsigned long long)((u >> 48) & 0x1f), (unsigned long long)((u >> 32) & 0x1f));
}

std::string block_path(const std::string& base, int64_t id) { return block_dir(base, id) + str_printf("/blk_%lld", (long long)id); }

static bool storage_from_name(const std::string& s, int32_t* t) {
    std::string u;
    for (char c : s) u.push_back(static_cast<char>(toupper(static_cast<unsigned char>(c))));
    if (u == "MEM") *t = kStorageMem;
    else if (u == "SSD") *t = kStorageSsd;
    else if (u == "HDD") *t = kStorageHdd;
    else if (u == "UFS") *t = kStorageUfs;
    else if (u == "DISK") *t = kStorageDisk;
    else return false;
    return true;
}

Err parse_data_dir(const std::string& spec, StorageDir* out) {
    *out = StorageDir();
    out->path = spec;
    if (spec.empty() || spec[0] != '[') return Err::ok();
    const size_t rb = spec.find(']');
    if (rb == std::string::npos || rb + 1 >= spec.size()) return Err::ok();
    const std::string prefix = spec.substr(1, rb - 1);
    if (prefix.empty()) return Err::ok();
    std::vector<std::string> arr;
    size_t p = 0;
    for (;;) {
        const size_t c = prefix.find(':', p);
        arr.push_back(prefix.substr(p, c == std::string::npos ? std::string::npos : c - p));
        if (c == std::string::npos) break;
        p = c + 1;
    }
    std::string type = "disk", cap = "0";
    int32_t t;
    if (arr.size() == 1) {
        if (storage_from_name(arr[0], &t)) type = arr[0];
        else cap = arr[0];
    } else if (arr.size() == 2) {
        type = arr[0], cap = arr[1];
    } else {
        return Err::common("Incorrect data format " + spec);
    }
    if (!storage_from_name(type, &t)) t = kStorageDisk;
    out->storage_type = t;
    CV_RETURN_IF_ERR(parse_byte_size(cap, &out->capacity));
    out->path = spec.substr(rb + 1);
    return Err::ok();
}

static Err mkdirs(const std::string& path) {
    std::string cur;
    for (size_t i = 0; i <= path.size(); i++) {
        if (i == path.size() || path[i] == '/') {
            if (!cur.empty() && mkdir(cur.c_str(), 0755) != 0 && errno != EEXIST) return Err::io(str_printf("mkdir %s: %s", cur.c_str(), strerror(errno)));
        }
        if (i < path.size()) cur.push_back(path[i]);
    }
    return Err::ok();
}

Err BlockStore::init(const std::vector<std::string>& data_dirs, const std::string& cluster_id, const ArenaOpts& arena) {
    dirs_.clear();
    blocks_.clear();
    size_t mem_dirs = 0;
    for (const auto& spec : data_dirs) {
        StorageDir d;
        CV_RETURN_IF_ERR(parse_data_dir(spec, &d));
        d.base_path = cluster_id.empty() ? d.path : d.path + "/" + cluster_id;
        CV_RETURN_IF_ERR(mkdirs(d.base_path + "/active"));
        if (arena.enable && d.storage_type == kStorageMem) {
            d.arena = std::make_shared<MemArena>();
            d.arena->reuse_delay_ms = arena.reuse_delay_ms;
            const int node = mem_dirs < arena.numa.size() ? arena.numa[mem_dirs] : -1;
            CV_RETURN_IF_ERR(d.arena->init(d.base_path + "/arena", d.capacity, arena.seg_bytes, node_cpus(node)));
            mem_dirs++;
        }
        CV_RETURN_IF_ERR(scan_dir(d));
        dirs_.push_back(d);
    }
    if (dirs_.empty()) return Err::common("worker.data_dir is empty");
    return Err::ok();
}

// vfs_dir.rs:339-362: the block map is rebuilt from file names and lengths
Err BlockStore::scan_dir(const StorageDir& d) {
    const std::string active = d.base_path + "/active";
    DIR* d1 = opendir(active.c_str());
    if (!d1) return Err::ok();
    while (dirent* e1 = readdir(d1)) {
        if (e1->d_name[0] != 'b') continue;
        const std::string p1 = active + "/" + e1->d_name;
        DIR* d2 = opendir(p1.c_str());
        if (!d2) continue;
        while (dirent* e2 = readdir(d2)) {
            if (e2->d_name[0] != 'b') continue;
            const std::string p2 = p1 + "/" + e2->d_name;
            DIR* d3 = opendir(p2.c_str());
            if (!d3) continue;
            while (dirent* e3 = readdir(d3)) {
                if (strncmp(e3->d_name, "blk_", 4) != 0) continue;
                char* end = nullptr;
                const long long id = strtoll(e3->d_name + 4, &end, 10);
                if (!end || *end) continue;
                struct stat st;
                const std::string fp = p2 + "/" + e3->d_name;
                if (stat(fp.c_str(), &st) != 0) continue;
                BlockMeta m;
                m.id = id, m.len = st.st_size, m.storage_type = d.storage_type, m.path = fp;
                if (d.arena && st.st_size < 128) {  // an extent descriptor, not block bytes
                    char text[128] = {0};
                    FILE* f = fopen(fp.c_str(), "r");
                    const size_t got = f ? fread(text, 1, sizeof(text) - 1, f) : 0;
                    if (f) fclose(f);
                    int64_t len = 0;
                    ArenaExtent ext;
                    if (got && MemArena::decode_descriptor(text, &ext, &len)) {
                        if (d.arena->mark_used(ext)) continue;  // stale descriptor (segment gone / overlap): not a block
                        m.len = len, m.hold = std::make_shared<ExtentHold>(d.arena, ext), m.path = d.arena->seg_path(ext.seg);
                    }
                }
                blocks_[id] = m;
            }
            closedir(d3);
        }
        closedir(d2);
    }
    closedir(d1);
    return Err::ok();
}

Err BlockStore::get_block(int64_t id, BlockMeta* out) const {
    std::lock_guard<std::mutex> lk(mu_);
    auto it = blocks_.find(id);
    if (it == blocks_.end()) return Err::common(str_printf("block %lld not exits", (long long)id));
    *out = it->second;
    return Err::ok();
}

size_t BlockStore::num_blocks() const {
    std::lock_guard<std::mutex> lk(mu_);
    return blocks_.size();
}

const StorageDir* BlockStore::choose_dir(int32_t storage_type, int dir_hint) {
    std::lock_guard<std::mutex> lk(mu_);
    std::vector<const StorageDir*> match, disk;
    for (const auto& d : dirs_) {
        if (d.storage_type == storage_type) match.push_back(&d);
        if (d.storage_type == kStorageDisk) disk.push_back(&d);
    }
    const auto& pool = !match.empty() ? match : disk;
    const size_t pick = dir_hint >= 0 ? static_cast<size_t>(dir_hint) : rr_++;
    if (pool.empty()) return dirs_.empty() ? nullptr : &dirs_[pick % dirs_.size()];
    return pool[pick % pool.size()];
}

Err BlockStore::register_meta(const BlockMeta& m) {
    std::shared_ptr<ExtentHold> old;  // the previous incarnation's extent is released outside the lock (when nobody reads it any more)
    std::lock_guard<std::mutex> lk(mu_);
    auto it = blocks_.find(m.id);
    if (it != blocks_.end()) old = std::move(it->second.hold);
    blocks_[m.id] = m;
    return Err::ok();
}

static Err write_descriptor(const std::string& stub, const ArenaExtent& e, int64_t len) {
    const std::string text = MemArena::encode_descriptor(e, len);
    const int fd = ::open(stub.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
    if (fd < 0) return Err::io(str_printf("open %s: %s", stub.c_str(), strerror(errno)));
    const ssize_t w = ::write(fd, text.data(), text.size());
    ::close(fd);
    if (w != static_cast<ssize_t>(text.size())) return Err::io(str_printf("write %s: %s", stub.c_str(), strerror(errno)));
    return Err::ok();
}

Err BlockStore::reserve_block(int64_t id, int64_t len, int32_t storage_type, int dir_hint, BlockWriteTarget* out) {
    const StorageDir* d = choose_dir(storage_type, dir_hint);
    if (!d) return Err::common("no storage dir");
    *out = BlockWriteTarget();
    out->dir_storage_type = d->storage_type;
    if (d->arena) {
        CV_RETURN_IF_ERR(d->arena->alloc(len, &out->ext));
        out->arena = d->arena;
        out->path = d->arena->seg_path(out->ext.seg);
        out->stub_path = block_path(d->base_path, id);
    } else {
        out->path = block_path(d->base_path, id);
    }
    Err e = mkdirs(block_dir(d->base_path, id));
    if (e && out->arena) out->arena->release_now(out->ext);
    return e;
}

Err BlockStore::open_block(int64_t id, int32_t storage_type, int64_t block_size, BlockWriteTarget* out) {
    BlockMeta old;
    bool had = false;
    {
        std::lock_guard<std::mutex> lk(mu_);
        auto wi = writing_.find(id);
        if (wi != writing_.end()) {  // already open (Open ... Complete arrive at different handler instances): the same extent
            *out = wi->second;
            return Err::ok();
        }
        auto it = blocks_.find(id);
        if (it != blocks_.end()) old = it->second, had = true;
    }
    if (had && !old.in_arena()) {  // re-opening an existing block writes to the same file
        *out = BlockWriteTarget();
        out->path = old.path, out->dir_storage_type = old.storage_type;
        return Err::ok();
    }
    if (had) {  // arena block: a fresh extent of block_size bytes with the old bytes in front; the old extent is released at commit
        const StorageDir* d = nullptr;
        for (const auto& x : dirs_)
            if (x.arena == old.hold->arena) d = &x;
        if (!d) return Err::common("arena of the block is gone");
        *out = BlockWriteTarget();
        CV_RETURN_IF_ERR(d->arena->alloc(std::max(block_size, old.len), &out->ext));
        out->arena = d->arena, out->path = d->arena->seg_path(out->ext.seg), out->dir_storage_type = old.storage_type;
        out->stub_path = block_path(d->base_path, id);
        memcpy(out->mem(), old.mem(), static_cast<size_t>(old.len));
        std::lock_guard<std::mutex> lk(mu_);
        writing_[id] = *out;
        return Err::ok();
    }
    CV_RETURN_IF_ERR(reserve_block(id, block_size, storage_type, -1, out));
    if (out->arena) {
        std::lock_guard<std::mutex> lk(mu_);
        writing_[id] = *out;
    }
    return Err::ok();
}

Err BlockStore::commit_block(int64_t id, BlockWriteTarget* t, int64_t len) {
    BlockMeta m;
    m.id = id, m.len = len, m.storage_type = t->dir_storage_type, m.path = t->path;
    if (t->arena) {
        {
            std::lock_guard<std::mutex> lk(mu_);
            writing_.erase(id);
        }
        if (len > t->ext.cap) return Err::common("committed length exceeds the reserved extent");
        t->arena->shrink(&t->ext, len);
        m.hold = std::make_shared<ExtentHold>(t->arena, t->ext);
        CV_RETURN_IF_ERR(write_descriptor(t->stub_path, t->ext, len));
    }
    return register_meta(m);
}

void BlockStore::abort_block(int64_t id, BlockWriteTarget* t) {
    if (t->arena) {
        {
            std::lock_guard<std::mutex> lk(mu_);
            writing_.erase(id);
        }
        t->arena->release_now(t->ext);  // never committed: nobody can be reading it
        t->ext = ArenaExtent();
        return;  // a previously committed incarnation (if any) stays as it was
    }
    ::unlink(t->path.c_str());
    std::lock_guard<std::mutex> lk(mu_);
    blocks_.erase(id);
}

void BlockStore::remove_block(int64_t id) {
    BlockMeta m;
    {
        std::lock_guard<std::mutex> lk(mu_);
        auto it = blocks_.find(id);
        if (it == blocks_.end()) return;
        m = it->second;
        blocks_.erase(it);
    }
    if (m.in_arena()) {
        for (const auto& d : dirs_)
            if (d.arena == m.hold->arena) ::unlink(block_path(d.base_path, id).c_str());
        // the extent itself goes back when the last reader's copy of the meta is gone (ExtentHold)
    } else {
        ::unlink(m.path.c_str());
    }
}

Err BlockStore::put_block(int64_t id, const void* data, int64_t len, int32_t storage_type, std::string* path_out, int dir_hint) {
    BlockWriteTarget t;
    CV_RETURN_IF_ERR(reserve_block(id, len, storage_type, dir_hint, &t));
    if (t.arena) {
        memcpy(t.mem(), data, static_cast<size_t>(len));
    } else {
        const int fd = ::open(t.path.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
        if (fd < 0) return Err::io(str_printf("open %s: %s", t.path.c_str(), strerror(errno)));
        const uint8_t* p = static_cast<const uint8_t*>(data);
        int64_t left = len;
        while (left > 0) {
            const ssize_t w = ::write(fd, p, static_cast<size_t>(left));
            if (w < 0) {
                if (errno == EINTR) continue;
                ::close(fd);
                return Err::io(str_printf("write %s: %s", t.path.c_str(), strerror(errno)));
            }
            p += w, left -= w;
        }
        ::close(fd);
    }
    if (path_out) *path_out = t.path;
    return commit_block(id, &t, len);
}

}  // namespace cv
