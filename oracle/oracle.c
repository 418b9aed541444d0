/*
 * oracle.c -- plain-C CPU restatement of the arithmetic on the Curvine sequential block-read path.
 *
 * TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): used by tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs as the checker or the timed CPU baseline; never
 * linked into or called by the product (curvine_b200/).
 *
 * What it restates (paths relative to the CurvineIO/curvine source tree):
 *   cvo_crc32 / cvo_crc32c      Utils::crc32 = crc32fast::hash        orpc/src/common/utils.rs:73-75
 *                               (crc32fast 1.4.2/1.5.0 is a crates.io dependency, absent from the tree:
 *                               restated from the published CRC-32/ISO-HDLC definition; pinned to the
 *                               check value 0xCBF43926 and to zlib in tests/test_oracle.py)
 *   cvo_bench_checksum          TaskResult::update_ck loop             curvine-tests/src/curvine_bench.rs:37-48,222-231
 *   cvo_synth_block             synthetic content generator            SURVEY.md §8(d) (ours; no reference counterpart)
 * The CPU *reader* restatement (per-chunk ping-pong client, short-circuit pread client) lives in
 * oracle/cpu_reader.c.
 */
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <stdlib.h>

#define POLY_IEEE 0xEDB88320u
#define POLY_CAST 0x82F63B78u

static uint32_t g_tab[2][8][256];
static int g_init;

static void init_tables(void) {
    if (g_init) return;
    const uint32_t polys[2] = {POLY_IEEE, POLY_CAST};
    for (int p = 0; p < 2; p++) {
        for (uint32_t i = 0; i < 256; i++) {
            uint32_t r = i;
            for (int k = 0; k < 8; k++) r = (r >> 1) ^ ((r & 1) ? polys[p] : 0);
            g_tab[p][0][i] = r;
        }
        for (uint32_t i = 0; i < 256; i++)
            for (int s = 1; s < 8; s++)
                g_tab[p][s][i] = (g_tab[p][s - 1][i] >> 8) ^ g_tab[p][0][g_tab[p][s - 1][i] & 0xff];
    }
    g_init = 1;
}

/* slicing-by-8, any of the two polynomials; crc is the running value (0 to start), zlib convention */
uint32_t cvo_crc(int poly_id, uint32_t crc, const uint8_t* buf, size_t len) {
    init_tables();
    uint32_t (*T)[256] = g_tab[poly_id ? 1 : 0];
    uint32_t r = ~crc;
    while (len && ((uintptr_t)buf & 7)) {
        r = T[0][(r ^ *buf++) & 0xff] ^ (r >> 8);
        len--;
    }
    while (len >= 8) {
        uint64_t w;
        memcpy(&w, buf, 8);
        uint32_t lo = (uint32_t)w ^ r, hi = (uint32_t)(w >> 32);
        r = T[7][lo & 0xff] ^ T[6][(lo >> 8) & 0xff] ^ T[5][(lo >> 16) & 0xff] ^ T[4][lo >> 24] ^
            T[3][hi & 0xff] ^ T[2][(hi >> 8) & 0xff] ^ T[1][(hi >> 16) & 0xff] ^ T[0][hi >> 24];
        buf += 8;
        len -= 8;
    }
    while (len--) r = T[0][(r ^ *buf++) & 0xff] ^ (r >> 8);
    return ~r;
}

/* bit-at-a-time definition (slow), the anchor the table versions are checked against */
uint32_t cvo_crc_bitwise(int poly_id, uint32_t crc, const uint8_t* buf, size_t len) {
    const uint32_t poly = poly_id ? POLY_CAST : POLY_IEEE;
    uint32_t r = ~crc;
    for (size_t i = 0; i < len; i++) {
        r ^= buf[i];
        for (int k = 0; k < 8; k++) r = (r >> 1) ^ ((r & 1) ? poly : 0);
    }
    return ~r;
}

uint32_t cvo_crc32(const uint8_t* buf, size_t len) { return cvo_crc(0, 0, buf, len); }
uint32_t cvo_crc32c(const uint8_t* buf, size_t len) { return cvo_crc(1, 0, buf, len); }

/* per-block CRCs of a buffer cut into block_size pieces */
void cvo_crc_blocks(int poly_id, const uint8_t* buf, size_t len, size_t block_size, uint32_t* out) {
    size_t b = 0;
    for (size_t pos = 0; pos < len; pos += block_size, b++) {
        size_t n = len - pos < block_size ? len - pos : block_size;
        out[b] = cvo_crc(poly_id, 0, buf + pos, n);
    }
}

/* curvine-bench read-side checksum: u64 sum of crc32 over every read buffer; the reference checksums the
 * whole buffer (&buf) even after a short final read (curvine_bench.rs:222-231) -> stale_tail != 0. */
uint64_t cvo_bench_checksum(const uint8_t* data, size_t len, size_t buf_size, int stale_tail) {
    uint8_t* buf = (uint8_t*)calloc(1, buf_size ? buf_size : 1);
    uint64_t sum = 0;
    for (size_t pos = 0; pos < len; pos += buf_size) {
        size_t n = len - pos < buf_size ? len - pos : buf_size;
        memcpy(buf, data + pos, n);
        sum += cvo_crc(0, 0, buf, stale_tail ? buf_size : n);
    }
    free(buf);
    return sum;
}

/* ---- synthetic content: xoshiro256** seeded by splitmix64(0xC0FFEEB200 ^ (file_id << 32) ^ block) ---- */
static inline uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }

void cvo_synth_block(uint64_t file_id, uint64_t block_index, uint8_t* out, size_t len) {
    uint64_t x = 0xC0FFEEB200ull ^ (file_id << 32) ^ block_index, s[4];
    for (int i = 0; i < 4; i++) {
        x += 0x9E3779B97F4A7C15ull;
        uint64_t z = x;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        s[i] = z ^ (z >> 31);
    }
    size_t pos = 0;
    while (pos < len) {
        const uint64_t r = rotl(s[1] * 5, 7) * 9, t = s[1] << 17;
        s[2] ^= s[0], s[3] ^= s[1], s[1] ^= s[2], s[0] ^= s[3], s[2] ^= t, s[3] = rotl(s[3], 45);
        size_t n = len - pos < 8 ? len - pos : 8;
        memcpy(out + pos, &r, n); /* little-endian host */
        pos += n;
    }
}
