/*
 * cpu_reader.c -- CPU restatement of the reference's sequential read path, kept structurally faithful.
 *
 * TEST INFRASTRUCTURE / CPU BASELINE ONLY (see oracle/__init__.py).  Never linked into the product.
 * The reference is Rust and cannot be built in this image; this port is what bench.py times as
 * cpu_baseline (kind "port") and as the `--impl reference` arm.
 *
 * Structure followed (paths relative to the CurvineIO/curvine source tree):
 *   caller loop     read_full(128 KiB buf) + Utils::crc32(buf) on the caller thread, u64 sum
 *                   curvine-tests/src/curvine_bench.rs:212-236,37-48
 *   Reader::read    one memcpy per byte out of the current chunk       curvine-common/src/fs/reader.rs:71-81
 *   prefetch        N sub-readers (N = read_parallel; smart prefetch: min(8, ceil(len/10 GiB))), slices of
 *                   read_slice_size striped slice_id % N, each with a bounded queue of read_chunk_num chunks
 *                   curvine-client/src/file/fs_reader_buffer.rs:147-222,332-406, fs_reader_parallel.rs:94-158,
 *                   read_detector.rs:130-135
 *   remote block    Open -> one synchronous Running request/response per read_chunk_size chunk -> Complete,
 *                   payload received into a heap buffer      block_reader_remote.rs:36-122, rpc_frame.rs:222-264
 *   local block     Open(short_circuit) -> pread read_chunk_size pieces of the block file -> Complete
 *                                                             block_reader_local.rs:43-143
 *   crc32           crc32fast (PCLMULQDQ folding on x86-64) -> restated here with PCLMUL 4x128-bit folding,
 *                   constants derived from x^n mod P at start-up and checked against the bitwise definition
 */
#include <arpa/inet.h>
#include <errno.h>
#include <fcntl.h>
#include <immintrin.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/socket.h>
#include <time.h>
#include <unistd.h>

uint32_t cvo_crc(int poly_id, uint32_t crc, const uint8_t* buf, size_t len);

/* ------------------------------------------------------------------ PCLMUL CRC-32 (IEEE) */
#define P_IEEE 0xEDB88320u
static uint32_t mulx(uint32_t a) { return (a >> 1) ^ ((a & 1) ? P_IEEE : 0); }
static uint32_t gfmul(uint32_t a, uint32_t b) {
    uint32_t r = 0;
    for (int i = 0; i < 32; i++) {
        if (b & (0x80000000u >> i)) r ^= a;
        a = mulx(a);
    }
    return r;
}
static uint32_t xpow(uint64_t n) {
    uint32_t r = 0x80000000u, b = 0x40000000u;
    while (n) {
        if (n & 1) r = gfmul(r, b);
        b = gfmul(b, b);
        n >>= 1;
    }
    return r;
}
static uint64_t k512_lo, k512_hi, k128_lo, k128_hi;
static int pcl_init;
static void pcl_setup(void) {
    if (pcl_init) return;
    /* clmul of two bit-reflected operands yields product * x; fold by D bits: lo qword * x^(D+64-33), hi * x^(D-33) */
    k512_lo = xpow(512 + 64 - 33), k512_hi = xpow(512 - 33);
    k128_lo = xpow(128 + 64 - 33), k128_hi = xpow(128 - 33);
    pcl_init = 1;
}
static inline __m128i fold(__m128i v, __m128i k, __m128i next) {
    return _mm_xor_si128(_mm_xor_si128(_mm_clmulepi64_si128(v, k, 0x00), _mm_clmulepi64_si128(v, k, 0x11)), next);
}

uint32_t cvo_crc32_pclmul(uint32_t crc, const uint8_t* buf, size_t len) {
    pcl_setup();
    if (len < 128) return cvo_crc(0, crc, buf, len);
    const __m128i k512 = _mm_set_epi64x((long long)k512_hi, (long long)k512_lo);
    const __m128i k128 = _mm_set_epi64x((long long)k128_hi, (long long)k128_lo);
    __m128i v0 = _mm_loadu_si128((const __m128i*)buf), v1 = _mm_loadu_si128((const __m128i*)(buf + 16));
    __m128i v2 = _mm_loadu_si128((const __m128i*)(buf + 32)), v3 = _mm_loadu_si128((const __m128i*)(buf + 48));
    v0 = _mm_xor_si128(v0, _mm_cvtsi32_si128((int)~crc)); /* init folded into the first 4 bytes */
    buf += 64, len -= 64;
    while (len >= 64) {
        v0 = fold(v0, k512, _mm_loadu_si128((const __m128i*)buf));
        v1 = fold(v1, k512, _mm_loadu_si128((const __m128i*)(buf + 16)));
        v2 = fold(v2, k512, _mm_loadu_si128((const __m128i*)(buf + 32)));
        v3 = fold(v3, k512, _mm_loadu_si128((const __m128i*)(buf + 48)));
        buf += 64, len -= 64;
    }
    v0 = fold(v0, k128, v1);
    v0 = fold(v0, k128, v2);
    v0 = fold(v0, k128, v3);
    while (len >= 16) {
        v0 = fold(v0, k128, _mm_loadu_si128((const __m128i*)buf));
        buf += 16, len -= 16;
    }
    uint8_t tmp[16];
    _mm_storeu_si128((__m128i*)tmp, v0);
    /* V(x) == M(x) mod P: run the 16 state bytes through the table from a zero register, then the tail.
     * cvo_crc(crc_in) starts its register at ~crc_in and returns ~register. */
    uint32_t r = cvo_crc(0, ~0u, tmp, 16);
    return cvo_crc(0, r, buf, len);
}

/* ------------------------------------------------------------------ tiny orpc client (22-byte big-endian prefix) */
static void be32(uint8_t* p, uint32_t v) { p[0] = v >> 24, p[1] = v >> 16, p[2] = v >> 8, p[3] = v; }
static void be64(uint8_t* p, uint64_t v) { be32(p, (uint32_t)(v >> 32)), be32(p + 4, (uint32_t)v); }
static uint32_t rd32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
static int send_all(int fd, const void* b, size_t n) {
    const uint8_t* p = b;
    while (n) {
        ssize_t w = send(fd, p, n, MSG_NOSIGNAL);
        if (w < 0) {
            if (errno == EINTR) continue;
            return -1;
        }
        p += w, n -= (size_t)w;
    }
    return 0;
}
static int recv_all(int fd, void* b, size_t n) {
    uint8_t* p = b;
    while (n) {
        ssize_t r = recv(fd, p, n, 0);
        if (r <= 0) {
            if (r < 0 && errno == EINTR) continue;
            return -1;
        }
        p += r, n -= (size_t)r;
    }
    return 0;
}
static size_t put_varint(uint8_t* p, uint64_t v) {
    size_t n = 0;
    while (v >= 0x80) p[n++] = (uint8_t)(v | 0x80), v >>= 7;
    p[n++] = (uint8_t)v;
    return n;
}
static size_t put_field(uint8_t* p, int no, int64_t v) {
    size_t n = put_varint(p, (uint64_t)no << 3);
    return n + put_varint(p + n, (uint64_t)v);
}
/* BlockReadRequest (worker.proto:38-47), all required fields in order */
static size_t enc_read_req(uint8_t* p, int64_t id, int64_t off, int64_t len, int32_t chunk, int sc, int ra, int64_t ra_len, int64_t drop) {
    size_t n = 0;
    n += put_field(p + n, 1, id), n += put_field(p + n, 2, off), n += put_field(p + n, 3, len), n += put_field(p + n, 4, chunk);
    n += put_field(p + n, 5, sc), n += put_field(p + n, 8, ra), n += put_field(p + n, 9, ra_len), n += put_field(p + n, 10, drop);
    return n;
}
static int rpc_send(int fd, int status, int64_t req_id, int32_t seq, const uint8_t* hdr, size_t hlen) {
    uint8_t b[22 + 128];
    be32(b, (uint32_t)(18 + hlen)), be32(b + 4, (uint32_t)hlen);
    b[8] = 81, b[9] = (uint8_t)(status | 0xF0);
    be64(b + 10, (uint64_t)req_id), be32(b + 18, (uint32_t)seq);
    if (hlen) memcpy(b + 22, hdr, hlen);
    return send_all(fd, b, 22 + hlen);
}
/* receive one response; header into hdr (cap 4096), payload into data (cap dcap); returns payload length or -1 */
static int64_t rpc_recv(int fd, int64_t req_id, int32_t seq, uint8_t* hdr, size_t* hlen, uint8_t* data, size_t dcap) {
    uint8_t p[22];
    if (recv_all(fd, p, 22)) return -1;
    int32_t total = (int32_t)rd32(p), hl = (int32_t)rd32(p + 4);
    int64_t dl = (int64_t)total - hl - 18;
    if (dl < 0 || dl > 16 * 1024 * 1024 || hl < 0 || hl > 4096) return -1;
    if (hl && recv_all(fd, hdr, (size_t)hl)) return -1;
    if ((size_t)dl > dcap) return -1;
    if (dl && recv_all(fd, data, (size_t)dl)) return -1;
    if (hlen) *hlen = (size_t)hl;
    int8_t st = (int8_t)p[9];
    uint64_t rid = ((uint64_t)rd32(p + 10) << 32) | rd32(p + 14);
    if ((st >> 4) != 0 || (int64_t)rid != req_id || (int32_t)rd32(p + 18) != seq) return -1; /* raw_client.rs:100-116 */
    return dl;
}
static int dial(const char* ip, int port) {
    int fd = socket(AF_INET, SOCK_STREAM, 0), one = 1;
    struct sockaddr_in sa;
    memset(&sa, 0, sizeof(sa));
    sa.sin_family = AF_INET, sa.sin_port = htons((uint16_t)port);
    inet_pton(AF_INET, ip, &sa.sin_addr);
    setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
    if (connect(fd, (struct sockaddr*)&sa, sizeof(sa))) {
        close(fd);
        return -1;
    }
    return fd;
}

/* ------------------------------------------------------------------ the reader */
typedef struct {
    int64_t off;
    size_t len;
    uint8_t* data;
} Chunk;

typedef struct {
    /* bounded mpsc of read_chunk_num chunks (fs_reader_buffer.rs:185-187) */
    Chunk* q;
    int cap, head, count, done, failed;
    pthread_mutex_t mu;
    pthread_cond_t not_empty, not_full;
} Queue;

typedef struct {
    const char* ip;
    int port, short_circuit;
    int64_t file_len, block_size, chunk_size, slice_size, limit;
    const int64_t* block_ids;
    int n_sub, sub_id;
    Queue* q;
} SubArgs;

static void q_push(Queue* q, Chunk c) {
    pthread_mutex_lock(&q->mu);
    while (q->count == q->cap) pthread_cond_wait(&q->not_full, &q->mu);
    q->q[(q->head + q->count++) % q->cap] = c;
    pthread_cond_signal(&q->not_empty);
    pthread_mutex_unlock(&q->mu);
}
static int q_pop(Queue* q, Chunk* c) {
    pthread_mutex_lock(&q->mu);
    while (q->count == 0 && !q->done) pthread_cond_wait(&q->not_empty, &q->mu);
    if (q->count == 0) {
        pthread_mutex_unlock(&q->mu);
        return 0;
    }
    *c = q->q[q->head];
    q->head = (q->head + 1) % q->cap, q->count--;
    pthread_cond_signal(&q->not_full);
    pthread_mutex_unlock(&q->mu);
    return 1;
}
static void q_finish(Queue* q, int failed) {
    pthread_mutex_lock(&q->mu);
    q->done = 1, q->failed |= failed;
    pthread_cond_broadcast(&q->not_empty);
    pthread_mutex_unlock(&q->mu);
}

/* one sub-reader: walks its slices; inside a slice, block by block, chunk by chunk */
static void* sub_reader(void* arg) {
    SubArgs* a = arg;
    int fd = dial(a->ip, a->port), failed = fd < 0;
    uint8_t hdr[4096], req[128];
    unsigned seed = 12345u + (unsigned)a->sub_id;
    const int64_t end_all = a->limit < a->file_len ? a->limit : a->file_len;
    int64_t n_slices = (a->file_len + a->slice_size - 1) / a->slice_size;
    for (int64_t s = a->sub_id; s < n_slices && !failed; s += a->n_sub) {
        int64_t pos = s * a->slice_size, send = pos + a->slice_size;
        if (a->n_sub == 1) pos = 0, send = a->file_len, s = n_slices; /* parallel 1: one slice (split(), :99-101) */
        if (send > end_all) send = end_all;
        while (pos < send && !failed) {
            /* a new BlockReader per (slice, block): handle cache is off for striped readers (fs_reader_parallel.rs:83-84) */
            const int64_t b = pos / a->block_size, boff = pos - b * a->block_size;
            int64_t blen = a->file_len - b * a->block_size;
            if (blen > a->block_size) blen = a->block_size;
            int64_t bend = boff + (send - pos);
            if (bend > blen) bend = blen;
            const int64_t req_id = (((int64_t)rand_r(&seed) << 31) ^ rand_r(&seed)) | ((int64_t)a->sub_id << 56);
            size_t hl = enc_read_req(req, a->block_ids[b], boff, blen, (int32_t)a->chunk_size, a->short_circuit, 1, a->chunk_size * 8, 1 << 20);
            size_t rhl = 0;
            if (rpc_send(fd, 2, req_id, 0, req, hl) || rpc_recv(fd, req_id, 0, hdr, &rhl, NULL, 0) < 0) {
                failed = 1;
                break;
            }
            int32_t seq = 0;
            int bfd = -1;
            if (a->short_circuit) {
                /* BlockReadResponse: field 3 = path */
                char path[2048] = {0};
                size_t i = 0;
                while (i < rhl) {
                    uint64_t key = 0, v = 0;
                    int sh = 0;
                    do key |= (uint64_t)(hdr[i] & 0x7f) << sh, sh += 7; while (hdr[i++] & 0x80);
                    sh = 0;
                    do v |= (uint64_t)(hdr[i] & 0x7f) << sh, sh += 7; while (hdr[i++] & 0x80);
                    if ((key & 7) == 2) {
                        if ((key >> 3) == 3 && v < sizeof(path)) memcpy(path, hdr + i, v);
                        i += v;
                    }
                }
                bfd = open(path, O_RDONLY);
                if (bfd < 0) failed = 1;
            }
            int64_t bp = boff;
            while (bp < bend && !failed) {
                int64_t want = blen - bp < a->chunk_size ? blen - bp : a->chunk_size;
                Chunk c = {b * a->block_size + bp, 0, malloc((size_t)want)}; /* fresh BytesMut per chunk */
                if (a->short_circuit) {
                    int64_t got = 0;
                    while (got < want) {
                        ssize_t r = pread(bfd, c.data + got, (size_t)(want - got), bp + got);
                        if (r <= 0) {
                            failed = 1;
                            break;
                        }
                        got += r;
                    }
                    c.len = (size_t)got;
                } else {
                    int64_t dl = -1;
                    if (!rpc_send(fd, 3, req_id, ++seq, NULL, 0)) dl = rpc_recv(fd, req_id, seq, hdr, NULL, c.data, (size_t)want);
                    if (dl != want) failed = 1;
                    c.len = (size_t)want;
                }
                if (failed) {
                    free(c.data);
                    break;
                }
                q_push(a->q, c);
                bp += want;
            }
            if (bfd >= 0) close(bfd);
            hl = enc_read_req(req, a->block_ids[b], 0, 0, 0, 0, 1, 4194304, 1048576);
            if (!failed && (rpc_send(fd, 5, req_id, seq + 1, req, hl) || rpc_recv(fd, req_id, seq + 1, hdr, NULL, NULL, 0) < 0)) failed = 1;
            pos += bend - boff;
        }
    }
    if (fd >= 0) close(fd);
    q_finish(a->q, failed);
    return NULL;
}

/*
 * Read [0, limit) of a file the way curvine-bench does and return the u64 sum of crc32 over buf_size buffers.
 * Returns 0 on success.  out[0] = bytes read, out[1] = checksum sum, out[2] = threads used (n_sub + 1).
 * use_pclmul: 1 = PCLMUL crc32 (crc32fast-class), 0 = slicing-by-8, -1 = no checksum.
 */
int cvo_cpu_read_file(const char* ip, int port, int short_circuit, int64_t file_len, int64_t block_size, const int64_t* block_ids,
                      int64_t chunk_size, int chunk_num, int read_parallel, int64_t buf_size, int64_t limit, int use_pclmul,
                      uint64_t out[3]) {
    if (limit <= 0 || limit > file_len) limit = file_len;
    const int64_t slice = chunk_size * chunk_num;
    int n_sub = read_parallel < 1 ? 1 : read_parallel;
    Queue* qs = calloc((size_t)n_sub, sizeof(Queue));
    SubArgs* as = calloc((size_t)n_sub, sizeof(SubArgs));
    pthread_t* th = calloc((size_t)n_sub, sizeof(pthread_t));
    for (int i = 0; i < n_sub; i++) {
        qs[i].cap = chunk_num, qs[i].q = calloc((size_t)chunk_num, sizeof(Chunk));
        pthread_mutex_init(&qs[i].mu, NULL), pthread_cond_init(&qs[i].not_empty, NULL), pthread_cond_init(&qs[i].not_full, NULL);
        as[i] = (SubArgs){ip, port, short_circuit, file_len, block_size, chunk_size, slice, limit, block_ids, n_sub, i, &qs[i]};
        pthread_create(&th[i], NULL, sub_reader, &as[i]);
    }
    uint8_t* buf = calloc(1, (size_t)buf_size);
    uint64_t sum = 0;
    int64_t pos = 0, filled = 0;
    Chunk cur = {0, 0, NULL};
    size_t cur_off = 0;
    int failed = 0;
    while (pos < limit && !failed) {
        if (cur_off >= cur.len) { /* FsReaderBuffer::read: pick the sub-reader that owns pos (fs_reader_buffer.rs:248-259) */
            free(cur.data);
            cur.data = NULL, cur.len = 0, cur_off = 0;
            Queue* q = &qs[(pos / slice) % n_sub];
            if (!q_pop(q, &cur) || cur.off != pos) {
                failed = 1;
                break;
            }
        }
        size_t n = cur.len - cur_off; /* Reader::read: memcpy out of the chunk (reader.rs:71-81) */
        if ((int64_t)n > buf_size - filled) n = (size_t)(buf_size - filled);
        if ((int64_t)n > limit - pos) n = (size_t)(limit - pos);
        memcpy(buf + filled, cur.data + cur_off, n);
        cur_off += n, filled += (int64_t)n, pos += (int64_t)n;
        if (filled == buf_size || pos == limit) { /* read_full returned: update_ck(&buf) over the whole buffer */
            if (use_pclmul > 0) sum += cvo_crc32_pclmul(0, buf, (size_t)buf_size);
            else if (use_pclmul == 0) sum += cvo_crc(0, 0, buf, (size_t)buf_size);
            filled = 0;
        }
    }
    free(cur.data);
    for (int i = 0; i < n_sub; i++) { /* drain so producers can finish */
        Chunk c;
        while (q_pop(&qs[i], &c)) free(c.data);
        pthread_join(th[i], NULL);
        failed |= qs[i].failed;
        free(qs[i].q);
    }
    free(qs), free(as), free(th), free(buf);
    out[0] = (uint64_t)pos, out[1] = sum, out[2] = (uint64_t)n_sub + 1;
    return failed ? -1 : 0;
}
