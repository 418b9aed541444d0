#include "wire.h"

#include <stdarg.h>
#include <stdio.h>
#include <time.h>

#include <atomic>
#include <random>

namespace cv {

std::string str_printf(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    return std::string(buf);
}

double now_sec() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec + ts.tv_nsec * 1e-9;
}

void encode_protocol(const Protocol& p, uint8_t out[kProtocolSize]) {
    put_be32(out, static_cast<uint32_t>(p.header_len + p.data_len + kHeadSize));
    put_be32(out + 4, static_cast<uint32_t>(p.header_len));
    out[8] = static_cast<uint8_t>(p.code);
    out[9] = static_cast<uint8_t>(status_encode(p.req_status, p.resp_status));
    put_be64(out + 10, static_cast<uint64_t>(p.req_id));
    put_be32(out + 18, static_cast<uint32_t>(p.seq_id));
}

Err decode_protocol(const uint8_t in[kProtocolSize], Protocol* p) {
    const int32_t total = static_cast<int32_t>(get_be32(in));
    const int32_t hsz = static_cast<int32_t>(get_be32(in + 4));
    const int64_t dsz = int64_t(total) - hsz - kHeadSize;
    if (dsz < 0) return Err::common("data length is negative");
    if (dsz > kMaxDataSize) return Err::common(str_printf("Data exceeds maximum size: %d", kMaxDataSize));
    p->code = static_cast<int8_t>(in[8]);
    status_decode(static_cast<int8_t>(in[9]), &p->req_status, &p->resp_status);
    p->req_id = static_cast<int64_t>(get_be64(in + 10));
    p->seq_id = static_cast<int32_t>(get_be32(in + 18));
    p->header_len = hsz;
    p->data_len = static_cast<int32_t>(dsz);
    return Err::ok();
}

Protocol request_proto(int8_t code, int8_t req_status, int64_t req_id, int32_t seq_id) {
    Protocol p;
    p.code = code, p.req_status = req_status, p.resp_status = kRespUndefined, p.req_id = req_id, p.seq_id = seq_id;
    return p;
}

// ---- proto2 as prost 0.11 writes it: required fields always present, in field order
static void put_varint(std::string* s, uint64_t v) {
    while (v >= 0x80) {
        s->push_back(static_cast<char>((v & 0x7f) | 0x80));
        v >>= 7;
    }
    s->push_back(static_cast<char>(v));
}
static void put_field(std::string* s, uint32_t no, int64_t v) {
    put_varint(s, uint64_t(no) << 3);
    put_varint(s, static_cast<uint64_t>(v));
}
static void put_bytes(std::string* s, uint32_t no, const std::string& b) {
    put_varint(s, (uint64_t(no) << 3) | 2);
    put_varint(s, b.size());
    s->append(b);
}

struct Field {
    uint32_t no;
    uint32_t wt;
    uint64_t v;
    const uint8_t* p;
    size_t n;
};

static bool get_varint(const uint8_t*& p, const uint8_t* end, uint64_t* v) {
    uint64_t r = 0;
    for (int shift = 0; shift < 70 && p < end; shift += 7) {
        const uint8_t b = *p++;
        r |= uint64_t(b & 0x7f) << shift;
        if (!(b & 0x80)) {
            *v = r;
            return true;
        }
    }
    return false;
}

static bool next_field(const uint8_t*& p, const uint8_t* end, Field* f) {
    uint64_t key;
    if (!get_varint(p, end, &key)) return false;
    f->no = static_cast<uint32_t>(key >> 3), f->wt = key & 7, f->v = 0, f->p = nullptr, f->n = 0;
    switch (f->wt) {
        case 0:
            return get_varint(p, end, &f->v);
        case 2: {
            uint64_t n;
            if (!get_varint(p, end, &n) || n > size_t(end - p)) return false;
            f->p = p, f->n = n, p += n;
            return true;
        }
        case 1:
            if (end - p < 8) return false;
            p += 8;
            return true;
        case 5:
            if (end - p < 4) return false;
            p += 4;
            return true;
        default:
            return false;
    }
}

std::string BlockReadRequest::encode() const {
    std::string s;
    put_field(&s, 1, id), put_field(&s, 2, off), put_field(&s, 3, len), put_field(&s, 4, chunk_size);
    put_field(&s, 5, short_circuit), put_field(&s, 8, enable_read_ahead), put_field(&s, 9, read_ahead_len);
    put_field(&s, 10, drop_cache_len);
    if (accept_arena) put_field(&s, 100, true);
    return s;
}

Err BlockReadRequest::decode(const uint8_t* p, size_t n, BlockReadRequest* o) {
    const uint8_t* end = p + n;
    uint32_t seen = 0;
    Field f;
    while (p < end) {
        if (!next_field(p, end, &f)) return Err(kPBDecode, "failed to decode BlockReadRequest");
        switch (f.no) {
            case 1: o->id = int64_t(f.v), seen |= 1; break;
            case 2: o->off = int64_t(f.v), seen |= 2; break;
            case 3: o->len = int64_t(f.v), seen |= 4; break;
            case 4: o->chunk_size = int32_t(f.v), seen |= 8; break;
            case 5: o->short_circuit = f.v != 0, seen |= 16; break;
            case 8: o->enable_read_ahead = f.v != 0, seen |= 32; break;
            case 9: o->read_ahead_len = int64_t(f.v), seen |= 64; break;
            case 10: o->drop_cache_len = int64_t(f.v), seen |= 128; break;
            case 100: o->accept_arena = f.v != 0; break;
            default: break;
        }
    }
    if (seen != 255) return Err(kPBDecode, "failed to decode BlockReadRequest: missing required field");
    return Err::ok();
}

std::string BlockReadResponse::encode() const {
    std::string s;
    put_field(&s, 1, id), put_field(&s, 2, len);
    if (has_path) put_bytes(&s, 3, path);
    put_field(&s, 4, storage_type);
    if (has_arena) put_field(&s, 100, arena_off), put_field(&s, 101, arena_seg_len);
    return s;
}

Err BlockReadResponse::decode(const uint8_t* p, size_t n, BlockReadResponse* o) {
    const uint8_t* end = p + n;
    uint32_t seen = 0;
    Field f;
    while (p < end) {
        if (!next_field(p, end, &f)) return Err(kPBDecode, "failed to decode BlockReadResponse");
        switch (f.no) {
            case 1: o->id = int64_t(f.v), seen |= 1; break;
            case 2: o->len = int64_t(f.v), seen |= 2; break;
            case 3: o->has_path = true, o->path.assign(reinterpret_cast<const char*>(f.p), f.n); break;
            case 4: o->storage_type = int32_t(f.v), seen |= 4; break;
            case 100: o->has_arena = true, o->arena_off = int64_t(f.v); break;
            case 101: o->arena_seg_len = int64_t(f.v); break;
            default: break;
        }
    }
    if (seen != 7) return Err(kPBDecode, "failed to decode BlockReadResponse: missing required field");
    return Err::ok();
}

std::string DataHeaderProto::encode() const {
    std::string s;
    put_field(&s, 1, offset), put_field(&s, 2, flush), put_field(&s, 3, is_last);
    return s;
}

Err DataHeaderProto::decode(const uint8_t* p, size_t n, DataHeaderProto* o) {
    const uint8_t* end = p + n;
    uint32_t seen = 0;
    Field f;
    while (p < end) {
        if (!next_field(p, end, &f)) return Err(kPBDecode, "failed to decode DataHeaderProto");
        switch (f.no) {
            case 1: o->offset = int64_t(f.v), seen |= 1; break;
            case 2: o->flush = f.v != 0, seen |= 2; break;
            case 3: o->is_last = f.v != 0, seen |= 4; break;
            default: break;
        }
    }
    if (seen != 7) return Err(kPBDecode, "failed to decode DataHeaderProto: missing required field");
    return Err::ok();
}

std::string BlockWriteRequest::encode() const {
    std::string b;
    put_field(&b, 1, block.id), put_field(&b, 2, block.block_size), put_field(&b, 3, block.storage_type), put_field(&b, 4, block.file_type);
    std::string s;
    put_bytes(&s, 1, b);
    put_field(&s, 2, off), put_field(&s, 3, block_size), put_field(&s, 4, short_circuit);
    put_bytes(&s, 5, client_name);
    put_field(&s, 6, chunk_size);
    return s;
}

Err BlockWriteRequest::decode(const uint8_t* p, size_t n, BlockWriteRequest* o) {
    const uint8_t* end = p + n;
    uint32_t seen = 0;
    Field f;
    while (p < end) {
        if (!next_field(p, end, &f)) return Err(kPBDecode, "failed to decode BlockWriteRequest");
        switch (f.no) {
            case 1: {
                const uint8_t* q = f.p;
                const uint8_t* qe = f.p + f.n;
                Field g;
                uint32_t bs = 0;
                while (q < qe) {
                    if (!next_field(q, qe, &g)) return Err(kPBDecode, "failed to decode ExtendedBlockProto");
                    if (g.no == 1) o->block.id = int64_t(g.v), bs |= 1;
                    else if (g.no == 2) o->block.block_size = int64_t(g.v), bs |= 2;
                    else if (g.no == 3) o->block.storage_type = int32_t(g.v), bs |= 4;
                    else if (g.no == 4) o->block.file_type = int32_t(g.v), bs |= 8;
                }
                if (bs != 15) return Err(kPBDecode, "failed to decode ExtendedBlockProto: missing required field");
                seen |= 1;
                break;
            }
            case 2: o->off = int64_t(f.v), seen |= 2; break;
            case 3: o->block_size = int64_t(f.v), seen |= 4; break;
            case 4: o->short_circuit = f.v != 0, seen |= 8; break;
            case 5: o->client_name.assign(reinterpret_cast<const char*>(f.p), f.n), seen |= 16; break;
            case 6: o->chunk_size = int32_t(f.v), seen |= 32; break;
            default: break;
        }
    }
    if (seen != 63) return Err(kPBDecode, "failed to decode BlockWriteRequest: missing required field");
    return Err::ok();
}

std::string BlockWriteResponse::encode() const {
    std::string s;
    put_field(&s, 1, id);
    if (has_path) put_bytes(&s, 2, path);
    put_field(&s, 3, off), put_field(&s, 4, block_size), put_field(&s, 5, storage_type);
    return s;
}

Err BlockWriteResponse::decode(const uint8_t* p, size_t n, BlockWriteResponse* o) {
    const uint8_t* end = p + n;
    uint32_t seen = 0;
    Field f;
    while (p < end) {
        if (!next_field(p, end, &f)) return Err(kPBDecode, "failed to decode BlockWriteResponse");
        switch (f.no) {
            case 1: o->id = int64_t(f.v), seen |= 1; break;
            case 2: o->has_path = true, o->path.assign(reinterpret_cast<const char*>(f.p), f.n); break;
            case 3: o->off = int64_t(f.v), seen |= 2; break;
            case 4: o->block_size = int64_t(f.v), seen |= 4; break;
            case 5: o->storage_type = int32_t(f.v), seen |= 8; break;
            default: break;
        }
    }
    if (seen != 15) return Err(kPBDecode, "failed to decode BlockWriteResponse: missing required field");
    return Err::ok();
}

std::string encode_error_body(int32_t kind, const std::string& msg) {
    std::string s(8, '\0');
    put_be32(reinterpret_cast<uint8_t*>(&s[0]), static_cast<uint32_t>(kind));
    put_be32(reinterpret_cast<uint8_t*>(&s[4]), static_cast<uint32_t>(msg.size()));
    s += msg;
    s.append(4, '\0');  // no attached data
    return s;
}

Err decode_error_body(const uint8_t* p, size_t n) {
    if (n < 8) return Err::common(std::string(reinterpret_cast<const char*>(p), n));
    const int32_t kind = static_cast<int32_t>(get_be32(p));
    size_t len = get_be32(p + 4);
    if (len > n - 8) len = n - 8;
    return Err(kind == 0 ? int32_t(kCommon) : kind, std::string(reinterpret_cast<const char*>(p + 8), len));
}

int64_t new_req_id() {
    static std::atomic<uint64_t> ctr{0};
    static const uint64_t seed = std::random_device{}();
    uint64_t x = seed + 0x9E3779B97F4A7C15ull * (ctr.fetch_add(1) + 1);
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    x ^= x >> 31;
    return static_cast<int64_t>(x & 0x7fffffffffffffffull);
}

}  // namespace cv
