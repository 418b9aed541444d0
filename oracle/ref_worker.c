/*
 * ref_worker.c -- a worker emulator for the reference arm of bench.py and for oracle-side tests.
 *
 * TEST INFRASTRUCTURE / CPU BASELINE ONLY (see oracle/__init__.py).  Never linked into the product; it exists so
 * that `bench.py --impl reference` times the oracle's CPU reader (cpu_reader.c) against something that is NOT the
 * product library.  It restates the worker side of the block-read path (paths relative to the CurvineIO/curvine source tree):
 *   BlockStore layout   <base>/active/b{(id>>48)&31}/b{(id>>32)&31}/blk_<id>, raw bytes
 *                       curvine-server/src/worker/block/block_meta.rs:199-237
 *   server loop         one stateful handler per connection, request -> handle -> response; errors become error responses
 *                       orpc/src/handler/stream_handler.rs:47-100, worker/handler/block_handler.rs:50-61
 *   ReadHandler         Open: look the block up, off <= len, chunk_size > 0, answer BlockReadResponse{id,len,path?,storage_type};
 *                       Running: optional DataHeaderProto seek, min(chunk, len-pos) bytes by sendfile; Complete
 *                       curvine-server/src/worker/handler/read_handler.rs:60-207
 *   frame               22-byte big-endian prefix  orpc/src/message/rpc_message.rs:301-338
 * Files are written by the oracle's own generator (oracle.c cvo_synth_block).
 */
#define _GNU_SOURCE
#include <arpa/inet.h>
#include <errno.h>
#include <fcntl.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/sendfile.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <unistd.h>

void cvo_synth_block(uint64_t file_id, uint64_t block_index, uint8_t* out, size_t len);

typedef struct RefWorker {
    char base[512];
    int lfd, port;
    volatile int stopping;
    pthread_t acc;
    pthread_mutex_t mu;
    int conns[1024];
    int nconns;
    volatile int live;
} RefWorker;

static void w_be32(uint8_t* p, uint32_t v) { p[0] = v >> 24, p[1] = v >> 16, p[2] = v >> 8, p[3] = v; }
static uint32_t r_be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }

static int tx(int fd, const void* b, size_t n, int more) {
    const uint8_t* p = b;
    while (n) {
        ssize_t w = send(fd, p, n, MSG_NOSIGNAL | (more ? MSG_MORE : 0));
        if (w < 0) {
            if (errno == EINTR) continue;
            return -1;
        }
        p += w, n -= (size_t)w;
    }
    return 0;
}
static int rx(int fd, void* b, size_t n) {
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
static size_t varint_put(uint8_t* p, uint64_t v) {
    size_t n = 0;
    while (v >= 0x80) p[n++] = (uint8_t)(v | 0x80), v >>= 7;
    p[n++] = (uint8_t)v;
    return n;
}
static int varint_get(const uint8_t** p, const uint8_t* end, uint64_t* v) {
    uint64_t r = 0;
    for (int s = 0; s < 70 && *p < end; s += 7) {
        uint8_t b = *(*p)++;
        r |= (uint64_t)(b & 0x7f) << s;
        if (!(b & 0x80)) {
            *v = r;
            return 0;
        }
    }
    return -1;
}

static void block_path(const RefWorker* w, int64_t id, char* out, size_t cap, int mk) {
    uint64_t u = (uint64_t)id;
    char dir[640];
    snprintf(dir, sizeof(dir), "%s/active/b%llu", w->base, (unsigned long long)((u >> 48) & 31));
    if (mk) mkdir(dir, 0755);
    snprintf(dir, sizeof(dir), "%s/active/b%llu/b%llu", w->base, (unsigned long long)((u >> 48) & 31), (unsigned long long)((u >> 32) & 31));
    if (mk) mkdir(dir, 0755);
    snprintf(out, cap, "%s/blk_%lld", dir, (long long)id);
}

/* response: prefix (+header) (+payload region of a file) */
static int respond(int fd, const uint8_t* req_prefix, int error, const uint8_t* header, int hlen, const uint8_t* data, int dlen, int file_fd, int64_t file_off,
                   int file_len) {
    uint8_t p[22];
    memcpy(p, req_prefix, 22);
    const int payload = file_fd >= 0 ? file_len : dlen;
    w_be32(p, (uint32_t)(18 + hlen + payload));
    w_be32(p + 4, (uint32_t)hlen);
    p[9] = (uint8_t)((req_prefix[9] & 0x0f) | (error ? 0x10 : 0x00));
    if (tx(fd, p, 22, hlen + payload > 0)) return -1;
    if (hlen && tx(fd, header, (size_t)hlen, payload > 0)) return -1;
    if (file_fd >= 0) {
        off_t o = file_off;
        size_t left = (size_t)file_len;
        while (left) {
            ssize_t s = sendfile(fd, file_fd, &o, left);
            if (s <= 0) {
                if (s < 0 && (errno == EINTR || errno == EAGAIN)) continue;
                return -1;
            }
            left -= (size_t)s;
        }
    } else if (dlen && tx(fd, data, (size_t)dlen, 0)) return -1;
    return 0;
}

static int respond_error(int fd, const uint8_t* req_prefix, const char* msg) {
    /* error_encoder.rs:24-51: i32 kind (Common = 10000) | i32 len | utf-8 message */
    uint8_t body[600];
    const size_t n = strlen(msg) > 500 ? 500 : strlen(msg);
    w_be32(body, 10000), w_be32(body + 4, (uint32_t)n);
    memcpy(body + 8, msg, n);
    return respond(fd, req_prefix, 1, NULL, 0, body, (int)(8 + n), -1, 0, 0);
}

static void* serve(void* arg) {
    void** a = arg;
    RefWorker* w = a[0];
    const int fd = (int)(intptr_t)a[1];
    free(arg);
    int bfd = -1;
    int64_t pos = 0, len = 0, chunk = 0;
    uint8_t prefix[22], header[256];
    for (;;) {
        if (rx(fd, prefix, 22)) break;
        const int hlen = (int)r_be32(prefix + 4), total = (int)r_be32(prefix);
        const int dlen = total - 18 - hlen;
        if (hlen < 0 || hlen > (int)sizeof(header) || dlen < 0) break;
        if (hlen && rx(fd, header, (size_t)hlen)) break;
        for (int left = dlen; left > 0;) { /* requests on the read path carry no payload; drain if any */
            uint8_t sink[256];
            int t = left > 256 ? 256 : left;
            if (rx(fd, sink, (size_t)t)) goto out;
            left -= t;
        }
        const int code = (int8_t)prefix[8], req_status = prefix[9] & 0x0f;
        if (req_status == 0) continue; /* heartbeat */
        if (code != 81) {
            if (respond_error(fd, prefix, "Unsupported request type")) break;
            continue;
        }
        if (req_status == 2) { /* Open: BlockReadRequest{1 id, 2 off, 3 len, 4 chunk_size, 5 short_circuit, ...} */
            int64_t id = 0, off = 0, csz = 0;
            int sc = 0;
            const uint8_t *p = header, *end = header + hlen;
            int bad = 0;
            while (p < end && !bad) {
                uint64_t key, v;
                if (varint_get(&p, end, &key) || (key & 7) != 0 || varint_get(&p, end, &v)) bad = 1;
                else if ((key >> 3) == 1) id = (int64_t)v;
                else if ((key >> 3) == 2) off = (int64_t)v;
                else if ((key >> 3) == 4) csz = (int64_t)v;
                else if ((key >> 3) == 5) sc = v != 0;
            }
            char path[768];
            block_path(w, id, path, sizeof(path), 0);
            struct stat st;
            if (bad || stat(path, &st) != 0) {
                char msg[128];
                snprintf(msg, sizeof(msg), "block %lld not exits", (long long)id);
                if (respond_error(fd, prefix, msg)) break;
                continue;
            }
            if (off > st.st_size || csz <= 0) {
                if (respond_error(fd, prefix, csz <= 0 ? "chunk_size must be greater than 0" : "The length of the requested data exceeds the maximum length of the block file")) break;
                continue;
            }
            if (bfd >= 0) close(bfd);
            bfd = -1;
            if (!sc) bfd = open(path, O_RDONLY | O_CLOEXEC);
            pos = off, len = st.st_size, chunk = csz;
            uint8_t h[900];
            size_t n = 0;
            h[n++] = 0x08, n += varint_put(h + n, (uint64_t)id);
            h[n++] = 0x10, n += varint_put(h + n, (uint64_t)len);
            if (sc) {
                const size_t pl = strlen(path);
                h[n++] = 0x1a, n += varint_put(h + n, pl);
                memcpy(h + n, path, pl), n += pl;
            }
            h[n++] = 0x20, h[n++] = 0; /* storage_type = MEM */
            if (respond(fd, prefix, 0, h, (int)n, NULL, 0, -1, 0, 0)) break;
        } else if (req_status == 3) { /* Running */
            if (bfd < 0) {
                if (respond_error(fd, prefix, "self.file is none")) break;
                continue;
            }
            if (hlen) { /* DataHeaderProto{1 offset,...}: seek */
                const uint8_t *p = header, *end = header + hlen;
                uint64_t key, v;
                while (p < end && !varint_get(&p, end, &key) && !varint_get(&p, end, &v))
                    if ((key >> 3) == 1) pos = (int64_t)v;
            }
            const int64_t c = chunk < len - pos ? chunk : len - pos;
            if (c <= 0) {
                if (respond_error(fd, prefix, "offset exceeds file length")) break;
                continue;
            }
            if (respond(fd, prefix, 0, NULL, 0, NULL, 0, bfd, pos, (int)c)) break;
            pos += c;
        } else if (req_status == 5 || req_status == 4) { /* Complete / Cancel */
            if (bfd >= 0) close(bfd);
            bfd = -1;
            if (respond(fd, prefix, 0, NULL, 0, NULL, 0, -1, 0, 0)) break;
        } else {
            if (respond_error(fd, prefix, "Unsupported request type")) break;
        }
    }
out:
    if (bfd >= 0) close(bfd);
    pthread_mutex_lock(&w->mu);
    for (int i = 0; i < w->nconns; i++)
        if (w->conns[i] == fd) {
            w->conns[i] = w->conns[--w->nconns];
            break;
        }
    pthread_mutex_unlock(&w->mu);
    close(fd);
    __sync_fetch_and_sub(&w->live, 1);
    return NULL;
}

static void* accept_loop(void* arg) {
    RefWorker* w = arg;
    while (!w->stopping) {
        int fd = accept(w->lfd, NULL, NULL);
        if (fd < 0) {
            if (errno == EINTR) continue;
            break;
        }
        int one = 1;
        setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
        pthread_mutex_lock(&w->mu);
        if (w->nconns >= 1024) {
            pthread_mutex_unlock(&w->mu);
            close(fd);
            continue;
        }
        w->conns[w->nconns++] = fd;
        pthread_mutex_unlock(&w->mu);
        __sync_fetch_and_add(&w->live, 1);
        void** a = malloc(2 * sizeof(void*));
        a[0] = w, a[1] = (void*)(intptr_t)fd;
        pthread_t t;
        pthread_attr_t at;
        pthread_attr_init(&at);
        pthread_attr_setdetachstate(&at, PTHREAD_CREATE_DETACHED);
        if (pthread_create(&t, &at, serve, a) != 0) {
            free(a);
            close(fd);
            __sync_fetch_and_sub(&w->live, 1);
        }
        pthread_attr_destroy(&at);
    }
    return NULL;
}

/* base = <data_dir>/<cluster_id>; returns NULL on failure; *port = the bound port */
void* cvo_ref_worker_start(const char* base, int* port) {
    RefWorker* w = calloc(1, sizeof(RefWorker));
    snprintf(w->base, sizeof(w->base), "%s", base);
    char d[640];
    mkdir(base, 0755);
    snprintf(d, sizeof(d), "%s/active", base);
    mkdir(d, 0755);
    pthread_mutex_init(&w->mu, NULL);
    w->lfd = socket(AF_INET, SOCK_STREAM, 0);
    int one = 1;
    setsockopt(w->lfd, SOL_SOCKET, SO_REUSEADDR, &one, sizeof(one));
    struct sockaddr_in a;
    memset(&a, 0, sizeof(a));
    a.sin_family = AF_INET, a.sin_addr.s_addr = htonl(INADDR_LOOPBACK), a.sin_port = 0;
    socklen_t al = sizeof(a);
    if (bind(w->lfd, (struct sockaddr*)&a, sizeof(a)) != 0 || listen(w->lfd, 256) != 0 || getsockname(w->lfd, (struct sockaddr*)&a, &al) != 0) {
        close(w->lfd);
        free(w);
        return NULL;
    }
    w->port = ntohs(a.sin_port);
    *port = w->port;
    pthread_create(&w->acc, NULL, accept_loop, w);
    return w;
}

void cvo_ref_worker_stop(void* h) {
    RefWorker* w = h;
    if (!w) return;
    w->stopping = 1;
    shutdown(w->lfd, SHUT_RDWR);
    pthread_join(w->acc, NULL);
    close(w->lfd);
    pthread_mutex_lock(&w->mu);
    for (int i = 0; i < w->nconns; i++) shutdown(w->conns[i], SHUT_RDWR);
    pthread_mutex_unlock(&w->mu);
    while (w->live > 0) usleep(1000);
    free(w);
}

typedef struct GenArg {
    RefWorker* w;
    int64_t inode, len, block_size, nb;
    volatile int64_t* next;
    volatile int* failed;
} GenArg;

static void* gen_thread(void* arg) {
    GenArg* g = arg;
    uint8_t* buf = malloc((size_t)g->block_size);
    for (;;) {
        const int64_t b = __sync_fetch_and_add(g->next, 1);
        if (b >= g->nb) break;
        const int64_t blen = g->block_size < g->len - b * g->block_size ? g->block_size : g->len - b * g->block_size;
        cvo_synth_block((uint64_t)g->inode, (uint64_t)b, buf, (size_t)blen);
        char path[768];
        block_path(g->w, ((g->inode & ((1ll << 40) - 1)) << 24) | b, path, sizeof(path), 1);
        const int fd = open(path, O_WRONLY | O_CREAT | O_TRUNC, 0644);
        if (fd < 0) {
            *g->failed = 1;
            break;
        }
        for (int64_t done = 0; done < blen;) {
            ssize_t wr = write(fd, buf + done, (size_t)(blen - done));
            if (wr <= 0) {
                if (wr < 0 && errno == EINTR) continue;
                *g->failed = 1;
                break;
            }
            done += wr;
        }
        close(fd);
    }
    free(buf);
    return NULL;
}

/* block b of file `inode` = generator block (inode, b), block_id = inode << 24 | b (inode_id.rs:48-60) */
int cvo_ref_worker_create_file(void* h, int64_t inode, int64_t len, int64_t block_size, int threads) {
    RefWorker* w = h;
    volatile int64_t next = 0;
    volatile int failed = 0;
    GenArg g = {w, inode, len, block_size, (len + block_size - 1) / block_size, &next, &failed};
    if (threads < 1) threads = 1;
    if (threads > 128) threads = 128;
    pthread_t ts[128];
    for (int t = 0; t < threads; t++) pthread_create(&ts[t], NULL, gen_thread, &g);
    for (int t = 0; t < threads; t++) pthread_join(ts[t], NULL);
    return failed ? -1 : 0;
}
