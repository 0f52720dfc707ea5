/*
 * randomx_oracle.c — CPU ORACLE for k2pow (RandomX).  TEST INFRASTRUCTURE ONLY (same rules as post_oracle.h).
 *
 * go-spacemesh's k2pow is "randomx-based proof of work" (cmd/root.go:254-259; RandomXMode
 * activation/post_types.go:116-121; the blocking RPC that asks the post-service for it activation/nipost.go:171;
 * the check inside Verify activation/post_verifier.go:150-160).  The arithmetic lives in post-rs (un-vendored,
 * Makefile-libs.Inc:49-51), which calls tevador/RandomX v1.1.x through the randomx-rs crate.  RandomX is not under
 * /root/reference, so this file restates the published RandomX specification (tevador/RandomX doc/specs.md):
 *   §3 primitives  Blake2b, Argon2d (v0x13), AesGenerator1R/4R, AesHash1R, SuperscalarHash
 *   §4 the virtual machine, §5 instruction set, §6 SuperscalarHash program generator, §7 cache/dataset.
 *
 * PARITY STATUS: pinned stage by stage (tests/test_randomx_oracle.py):
 *   Blake2b          == hashlib.blake2b
 *   Argon2d fill     tag of the filled memory == cryptography's Argon2d (OpenSSL) with the same parameters
 *   AES generators   keys / initial states reproduce their published derivation (Blake2b of fixed ASCII strings),
 *                    single rounds == AES-NI
 *   whole function   RandomX's own known-answer vectors (src/tests/tests.cpp): key "test key 000",
 *                    input "This is a test" -> 639183aa...0b4e3f, and four more.  A 256-bit match of the final
 *                    hash pins every stage in between (cache, SuperscalarHash, dataset items, VM).
 *   The k2pow INPUT LAYOUT (pow[0:7] || nonce_group || challenge[0:8] || node_id, cache key string, difficulty
 *   scaling) is a recollection of post-rs with no fixture in the reference tree: "parity unpinned".
 */
#define _GNU_SOURCE
#include "randomx_oracle.h"

#include <emmintrin.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef __AES__
#include <wmmintrin.h>
#endif

/* ------------------------------------------------------------------------------------------------ */
/* Blake2b (RFC 7693), unkeyed                                                                      */
/* ------------------------------------------------------------------------------------------------ */
static const uint64_t B2B_IV[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL,
                                   0xa54ff53a5f1d36f1ULL, 0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL,
                                   0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
static const uint8_t B2B_SIGMA[12][16] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
    {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
    {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
    {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
    {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};

static inline uint64_t rotr64(uint64_t x, unsigned c) { return (x >> (c & 63)) | (x << ((64 - c) & 63)); }
static inline uint64_t rotl64(uint64_t x, unsigned c) { return (x << (c & 63)) | (x >> ((64 - c) & 63)); }
static inline uint64_t load64(const void *p) { uint64_t v; memcpy(&v, p, 8); return v; }
static inline uint32_t load32(const void *p) { uint32_t v; memcpy(&v, p, 4); return v; }
static inline void store64(void *p, uint64_t v) { memcpy(p, &v, 8); }
static inline void store32(void *p, uint32_t v) { memcpy(p, &v, 4); }

typedef struct { uint64_t h[8], t[2]; uint8_t buf[128]; size_t buflen, outlen; } b2b_state;

static void b2b_compress(b2b_state *S, const uint8_t block[128], int last) {
    uint64_t m[16], v[16];
    for (int i = 0; i < 16; i++) m[i] = load64(block + 8 * i);
    for (int i = 0; i < 8; i++) { v[i] = S->h[i]; v[i + 8] = B2B_IV[i]; }
    v[12] ^= S->t[0]; v[13] ^= S->t[1];
    if (last) v[14] = ~v[14];
#define B2G(r, i, a, b, c, d)                                  \
    a = a + b + m[B2B_SIGMA[r][2 * i]];     d = rotr64(d ^ a, 32); \
    c = c + d;                              b = rotr64(b ^ c, 24); \
    a = a + b + m[B2B_SIGMA[r][2 * i + 1]]; d = rotr64(d ^ a, 16); \
    c = c + d;                              b = rotr64(b ^ c, 63);
    for (int r = 0; r < 12; r++) {
        B2G(r, 0, v[0], v[4], v[8], v[12]) B2G(r, 1, v[1], v[5], v[9], v[13])
        B2G(r, 2, v[2], v[6], v[10], v[14]) B2G(r, 3, v[3], v[7], v[11], v[15])
        B2G(r, 4, v[0], v[5], v[10], v[15]) B2G(r, 5, v[1], v[6], v[11], v[12])
        B2G(r, 6, v[2], v[7], v[8], v[13]) B2G(r, 7, v[3], v[4], v[9], v[14])
    }
#undef B2G
    for (int i = 0; i < 8; i++) S->h[i] ^= v[i] ^ v[i + 8];
}
static void b2b_init(b2b_state *S, size_t outlen) {
    memset(S, 0, sizeof *S);
    for (int i = 0; i < 8; i++) S->h[i] = B2B_IV[i];
    S->h[0] ^= 0x01010000ULL ^ (uint64_t)outlen;
    S->outlen = outlen;
}
static void b2b_update(b2b_state *S, const void *in_, size_t inlen) {
    const uint8_t *in = (const uint8_t *)in_;
    while (inlen > 0) {
        if (S->buflen == 128) {   /* buffer full and more input follows: compress as a non-final block */
            S->t[0] += 128; if (S->t[0] < 128) S->t[1]++;
            b2b_compress(S, S->buf, 0);
            S->buflen = 0;
        }
        size_t take = 128 - S->buflen; if (take > inlen) take = inlen;
        memcpy(S->buf + S->buflen, in, take);
        S->buflen += take; in += take; inlen -= take;
    }
}
static void b2b_final(b2b_state *S, void *out) {
    S->t[0] += S->buflen; if (S->t[0] < S->buflen) S->t[1]++;
    memset(S->buf + S->buflen, 0, 128 - S->buflen);
    b2b_compress(S, S->buf, 1);
    uint8_t full[64];
    for (int i = 0; i < 8; i++) store64(full + 8 * i, S->h[i]);
    memcpy(out, full, S->outlen);
}
void rxo_blake2b(void *out, size_t outlen, const void *in, size_t inlen) {
    b2b_state S; b2b_init(&S, outlen); b2b_update(&S, in, inlen); b2b_final(&S, out);
}

/* ------------------------------------------------------------------------------------------------ */
/* Argon2d v0x13, single lane (RandomX spec §7.1: the cache is the Argon2d memory itself)            */
/* ------------------------------------------------------------------------------------------------ */
static void argon2_hprime(uint8_t *out, uint32_t outlen, const uint8_t *in, size_t inlen) {
    uint8_t le[4]; store32(le, outlen);
    b2b_state S;
    if (outlen <= 64) { b2b_init(&S, outlen); b2b_update(&S, le, 4); b2b_update(&S, in, inlen); b2b_final(&S, out); return; }
    uint8_t v[64], w[64];
    b2b_init(&S, 64); b2b_update(&S, le, 4); b2b_update(&S, in, inlen); b2b_final(&S, v);
    memcpy(out, v, 32); out += 32;
    uint32_t togo = outlen - 32;
    while (togo > 64) { rxo_blake2b(w, 64, v, 64); memcpy(v, w, 64); memcpy(out, v, 32); out += 32; togo -= 32; }
    rxo_blake2b(w, togo, v, 64);
    memcpy(out, w, togo);
}
static inline uint64_t blamka(uint64_t x, uint64_t y) { return x + y + 2 * (uint64_t)(uint32_t)x * (uint64_t)(uint32_t)y; }
#define AG(a, b, c, d)                                   \
    a = blamka(a, b); d = rotr64(d ^ a, 32); c = blamka(c, d); b = rotr64(b ^ c, 24); \
    a = blamka(a, b); d = rotr64(d ^ a, 16); c = blamka(c, d); b = rotr64(b ^ c, 63);
#define AROUND(v0, v1, v2, v3, v4, v5, v6, v7, v8, v9, v10, v11, v12, v13, v14, v15) \
    AG(v0, v4, v8, v12) AG(v1, v5, v9, v13) AG(v2, v6, v10, v14) AG(v3, v7, v11, v15) \
    AG(v0, v5, v10, v15) AG(v1, v6, v11, v12) AG(v2, v7, v8, v13) AG(v3, v4, v9, v14)
static void argon2_fill_block(const uint64_t *prev, const uint64_t *ref, uint64_t *next, int with_xor) {
    uint64_t R[128], T[128];
    for (int i = 0; i < 128; i++) { R[i] = prev[i] ^ ref[i]; T[i] = with_xor ? (R[i] ^ next[i]) : R[i]; }
    for (int i = 0; i < 8; i++) {
        uint64_t *v = R + 16 * i;
        AROUND(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7], v[8], v[9], v[10], v[11], v[12], v[13], v[14], v[15])
    }
    for (int i = 0; i < 8; i++) {
        uint64_t *v = R + 2 * i;
        AROUND(v[0], v[1], v[16], v[17], v[32], v[33], v[48], v[49], v[64], v[65], v[80], v[81], v[96], v[97], v[112], v[113])
    }
    for (int i = 0; i < 128; i++) next[i] = T[i] ^ R[i];
}
/* Fills `mem` (m_blocks x 1024 bytes, m_blocks a multiple of 4) as Argon2d with one lane; writes the taglen-byte
 * tag to `tag` if taglen > 0 (RandomX itself uses taglen = 0 and reads the memory). */
int rxo_argon2d_fill(uint64_t *mem, uint32_t m_blocks, uint32_t t_cost, const void *pwd, uint32_t pwdlen,
                     const void *salt, uint32_t saltlen, uint32_t taglen, uint8_t *tag) {
    if (m_blocks < 8 || (m_blocks & 3) || t_cost < 1) return -1;
    uint8_t h0[72], le[4];
    b2b_state S; b2b_init(&S, 64);
    uint32_t hdr[6] = {1 /*lanes*/, taglen, m_blocks /*m_cost in KiB*/, t_cost, 0x13, 0 /*Argon2d*/};
    for (int i = 0; i < 6; i++) { store32(le, hdr[i]); b2b_update(&S, le, 4); }
    store32(le, pwdlen); b2b_update(&S, le, 4); b2b_update(&S, pwd, pwdlen);
    store32(le, saltlen); b2b_update(&S, le, 4); b2b_update(&S, salt, saltlen);
    store32(le, 0); b2b_update(&S, le, 4); b2b_update(&S, le, 4);   /* no secret, no associated data */
    b2b_final(&S, h0);
    store32(h0 + 68, 0);                                   /* lane 0 */
    store32(h0 + 64, 0); argon2_hprime((uint8_t *)mem, 1024, h0, 72);
    store32(h0 + 64, 1); argon2_hprime((uint8_t *)(mem + 128), 1024, h0, 72);
    const uint32_t lane_len = m_blocks, seg = m_blocks / 4;
    for (uint32_t pass = 0; pass < t_cost; pass++)
        for (uint32_t slice = 0; slice < 4; slice++)
            for (uint32_t idx = (pass == 0 && slice == 0) ? 2 : 0; idx < seg; idx++) {
                uint32_t cur = slice * seg + idx;
                uint32_t prev = cur == 0 ? lane_len - 1 : cur - 1;
                uint64_t j1 = mem[(size_t)prev * 128] & 0xffffffffULL;
                uint32_t area = pass == 0 ? (slice * seg + idx - 1) : (lane_len - seg + idx - 1);
                uint64_t rel = (j1 * j1) >> 32;
                rel = area - 1 - ((area * rel) >> 32);
                uint32_t startp = (pass != 0 && slice != 3) ? (slice + 1) * seg : 0;
                uint32_t refi = (uint32_t)((startp + rel) % lane_len);
                argon2_fill_block(mem + (size_t)prev * 128, mem + (size_t)refi * 128, mem + (size_t)cur * 128, pass != 0);
            }
    if (taglen && tag) argon2_hprime(tag, taglen, (const uint8_t *)(mem + (size_t)(lane_len - 1) * 128), 1024);
    return 0;
}

/* ------------------------------------------------------------------------------------------------ */
/* AES single rounds (x86 AESENC / AESDEC semantics), portable + AES-NI                               */
/* ------------------------------------------------------------------------------------------------ */
static uint8_t SBOX[256], INV_SBOX[256];
static int g_tables_ready;
static uint8_t gmul(uint8_t a, uint8_t b) {
    uint8_t p = 0;
    for (int i = 0; i < 8; i++) { if (b & 1) p ^= a; uint8_t hi = a & 0x80; a <<= 1; if (hi) a ^= 0x1b; b >>= 1; }
    return p;
}
static void aes_tables(void) {
    if (g_tables_ready) return;
    /* multiplicative inverse via exponentiation table of generator 3, then the affine map (FIPS-197 §5.1.1) */
    uint8_t p = 1, q = 1;
    do {
        p = p ^ (uint8_t)(p << 1) ^ ((p & 0x80) ? 0x1b : 0);
        q ^= q << 1; q ^= q << 2; q ^= q << 4; if (q & 0x80) q ^= 0x09;
        uint8_t x = q ^ (uint8_t)((q << 1) | (q >> 7)) ^ (uint8_t)((q << 2) | (q >> 6)) ^ (uint8_t)((q << 3) | (q >> 5)) ^
                    (uint8_t)((q << 4) | (q >> 4));
        SBOX[p] = x ^ 0x63;
    } while (p != 1);
    SBOX[0] = 0x63;
    for (int i = 0; i < 256; i++) INV_SBOX[SBOX[i]] = (uint8_t)i;
    __sync_synchronize();
    g_tables_ready = 1;
}
void rxo_soft_aesenc(uint8_t st[16], const uint8_t key[16]) {
    aes_tables();
    uint8_t t[16];
    for (int c = 0; c < 4; c++) for (int r = 0; r < 4; r++) t[4 * c + r] = SBOX[st[4 * ((c + r) & 3) + r]];   /* SubBytes + ShiftRows */
    for (int c = 0; c < 4; c++) {
        const uint8_t *a = t + 4 * c;
        st[4 * c + 0] = gmul(a[0], 2) ^ gmul(a[1], 3) ^ a[2] ^ a[3] ^ key[4 * c + 0];
        st[4 * c + 1] = a[0] ^ gmul(a[1], 2) ^ gmul(a[2], 3) ^ a[3] ^ key[4 * c + 1];
        st[4 * c + 2] = a[0] ^ a[1] ^ gmul(a[2], 2) ^ gmul(a[3], 3) ^ key[4 * c + 2];
        st[4 * c + 3] = gmul(a[0], 3) ^ a[1] ^ a[2] ^ gmul(a[3], 2) ^ key[4 * c + 3];
    }
}
void rxo_soft_aesdec(uint8_t st[16], const uint8_t key[16]) {
    aes_tables();
    uint8_t t[16];
    for (int c = 0; c < 4; c++) for (int r = 0; r < 4; r++) t[4 * c + r] = INV_SBOX[st[4 * ((c - r) & 3) + r]];   /* InvShiftRows + InvSubBytes */
    for (int c = 0; c < 4; c++) {
        const uint8_t *a = t + 4 * c;
        st[4 * c + 0] = gmul(a[0], 14) ^ gmul(a[1], 11) ^ gmul(a[2], 13) ^ gmul(a[3], 9) ^ key[4 * c + 0];
        st[4 * c + 1] = gmul(a[0], 9) ^ gmul(a[1], 14) ^ gmul(a[2], 11) ^ gmul(a[3], 13) ^ key[4 * c + 1];
        st[4 * c + 2] = gmul(a[0], 13) ^ gmul(a[1], 9) ^ gmul(a[2], 14) ^ gmul(a[3], 11) ^ key[4 * c + 2];
        st[4 * c + 3] = gmul(a[0], 11) ^ gmul(a[1], 13) ^ gmul(a[2], 9) ^ gmul(a[3], 14) ^ key[4 * c + 3];
    }
}
static int g_soft_aes = 0;
void rxo_set_soft_aes(int on) { g_soft_aes = on; }
int rxo_has_aesni(void) {
#ifdef __AES__
    return __builtin_cpu_supports("aes") ? 1 : 0;
#else
    return 0;
#endif
}
static inline void aesenc(uint8_t st[16], const uint8_t key[16]) {
#ifdef __AES__
    if (!g_soft_aes) {
        _mm_storeu_si128((__m128i *)st, _mm_aesenc_si128(_mm_loadu_si128((const __m128i *)st), _mm_loadu_si128((const __m128i *)key)));
        return;
    }
#endif
    rxo_soft_aesenc(st, key);
}
static inline void aesdec(uint8_t st[16], const uint8_t key[16]) {
#ifdef __AES__
    if (!g_soft_aes) {
        _mm_storeu_si128((__m128i *)st, _mm_aesdec_si128(_mm_loadu_si128((const __m128i *)st), _mm_loadu_si128((const __m128i *)key)));
        return;
    }
#endif
    rxo_soft_aesdec(st, key);
}

/* Generator / hash constants (spec §3.2-3.4): Blake2b of fixed strings, derived once at start-up. */
static uint8_t GEN1R_KEYS[64], GEN4R_KEYS[128], HASH1R_STATE[64], HASH1R_XKEYS[32];
static int g_consts_ready;
static pthread_mutex_t g_init_mu = PTHREAD_MUTEX_INITIALIZER;
static void rx_consts(void) {
    if (g_consts_ready) return;
    pthread_mutex_lock(&g_init_mu);
    if (!g_consts_ready) {
        aes_tables();
        rxo_blake2b(GEN1R_KEYS, 64, "RandomX AesGenerator1R keys", 27);
        rxo_blake2b(GEN4R_KEYS, 64, "RandomX AesGenerator4R keys 0-3", 31);
        rxo_blake2b(GEN4R_KEYS + 64, 64, "RandomX AesGenerator4R keys 4-7", 31);
        rxo_blake2b(HASH1R_STATE, 64, "RandomX AesHash1R state", 23);
        rxo_blake2b(HASH1R_XKEYS, 32, "RandomX AesHash1R xkeys", 23);
        __sync_synchronize();
        g_consts_ready = 1;
    }
    pthread_mutex_unlock(&g_init_mu);
}
void rxo_aes_constants(uint8_t gen1r[64], uint8_t gen4r[128], uint8_t hash_state[64], uint8_t hash_xkeys[32]) {
    rx_consts();
    memcpy(gen1r, GEN1R_KEYS, 64); memcpy(gen4r, GEN4R_KEYS, 128); memcpy(hash_state, HASH1R_STATE, 64); memcpy(hash_xkeys, HASH1R_XKEYS, 32);
}
/* AesGenerator1R (spec §3.2): state columns 0,2 decrypt, 1,3 encrypt; output = the new state; state written back. */
void rxo_fill_aes_1rx4(uint8_t state[64], size_t outlen, uint8_t *out) {
    rx_consts();
    for (size_t off = 0; off < outlen; off += 64) {
        aesdec(state + 0, GEN1R_KEYS + 0); aesenc(state + 16, GEN1R_KEYS + 16);
        aesdec(state + 32, GEN1R_KEYS + 32); aesenc(state + 48, GEN1R_KEYS + 48);
        memcpy(out + off, state, 64);
    }
}
/* AesGenerator4R (spec §3.3): four rounds per output; columns 0,1 use keys 0-3, columns 2,3 keys 4-7. */
void rxo_fill_aes_4rx4(const uint8_t state_in[64], size_t outlen, uint8_t *out) {
    rx_consts();
    uint8_t st[64]; memcpy(st, state_in, 64);
    for (size_t off = 0; off < outlen; off += 64) {
        for (int k = 0; k < 4; k++) {
            aesdec(st + 0, GEN4R_KEYS + 16 * k); aesenc(st + 16, GEN4R_KEYS + 16 * k);
            aesdec(st + 32, GEN4R_KEYS + 64 + 16 * k); aesenc(st + 48, GEN4R_KEYS + 64 + 16 * k);
        }
        memcpy(out + off, st, 64);
    }
}
/* AesHash1R (spec §3.4): input blocks are the round keys; columns 0,2 encrypt, 1,3 decrypt; two finishing rounds. */
void rxo_hash_aes_1rx4(const uint8_t *in, size_t inlen, uint8_t out[64]) {
    rx_consts();
    uint8_t st[64]; memcpy(st, HASH1R_STATE, 64);
    for (size_t off = 0; off < inlen; off += 64) {
        aesenc(st + 0, in + off); aesdec(st + 16, in + off + 16); aesenc(st + 32, in + off + 32); aesdec(st + 48, in + off + 48);
    }
    for (int k = 0; k < 2; k++) {
        aesenc(st + 0, HASH1R_XKEYS + 16 * k); aesdec(st + 16, HASH1R_XKEYS + 16 * k);
        aesenc(st + 32, HASH1R_XKEYS + 16 * k); aesdec(st + 48, HASH1R_XKEYS + 16 * k);
    }
    memcpy(out, st, 64);
}

/* ------------------------------------------------------------------------------------------------ */
/* SuperscalarHash (spec §6): program generator simulating a 3-port superscalar CPU + executor        */
/* ------------------------------------------------------------------------------------------------ */
enum { SS_ISUB_R = 0, SS_IXOR_R, SS_IADD_RS, SS_IMUL_R, SS_IROR_C, SS_IADD_C7, SS_IXOR_C7, SS_IADD_C8, SS_IXOR_C8,
       SS_IADD_C9, SS_IXOR_C9, SS_IMULH_R, SS_ISMULH_R, SS_IMUL_RCP, SS_COUNT, SS_INVALID = -1 };
#define SS_LATENCY 170
#define SS_MAXSIZE (3 * SS_LATENCY + 2)
#define CYCLE_MAP (SS_LATENCY + 4)
#define LOOK_FORWARD 4
#define MAX_THROWAWAY 256
#define REG_NEEDS_DISP 5
enum { P0 = 1, P1 = 2, P5 = 4, P01 = 3, P05 = 5, P015 = 7 };

typedef struct { int size, latency, uop1, uop2, dependent; } macro_op;
/* macro-ops (spec table 6.2.1) */
static const macro_op M_SUB_RR = {3, 1, P015, 0, 0}, M_XOR_RR = {3, 1, P015, 0, 0}, M_IMUL_R = {3, 4, P1, P5, 0},
                      M_MUL_R = {3, 4, P1, P5, 0}, M_MOV_RR = {3, 0, 0, 0, 0}, M_MOV_RR_DEP = {3, 0, 0, 0, 1},
                      M_LEA_SIB = {4, 1, P01, 0, 0}, M_IMUL_RR = {4, 3, P1, 0, 0}, M_IMUL_RR_DEP = {4, 3, P1, 0, 1},
                      M_ROR_RI = {4, 1, P05, 0, 0}, M_ADD_RI = {7, 1, P015, 0, 0}, M_XOR_RI = {7, 1, P015, 0, 0},
                      M_MOV_RI64 = {10, 1, P015, 0, 0};
typedef struct { int type, nops; macro_op ops[3]; int result_op, dst_op, src_op; } ss_info;
static const ss_info SS_INFO[SS_COUNT] = {
    {SS_ISUB_R, 1, {M_SUB_RR}, 0, 0, 0},   {SS_IXOR_R, 1, {M_XOR_RR}, 0, 0, 0},   {SS_IADD_RS, 1, {M_LEA_SIB}, 0, 0, 0},
    {SS_IMUL_R, 1, {M_IMUL_RR}, 0, 0, 0},  {SS_IROR_C, 1, {M_ROR_RI}, 0, 0, -1},  {SS_IADD_C7, 1, {M_ADD_RI}, 0, 0, -1},
    {SS_IXOR_C7, 1, {M_XOR_RI}, 0, 0, -1}, {SS_IADD_C8, 1, {M_ADD_RI}, 0, 0, -1}, {SS_IXOR_C8, 1, {M_XOR_RI}, 0, 0, -1},
    {SS_IADD_C9, 1, {M_ADD_RI}, 0, 0, -1}, {SS_IXOR_C9, 1, {M_XOR_RI}, 0, 0, -1},
    {SS_IMULH_R, 3, {M_MOV_RR, M_MUL_R, M_MOV_RR_DEP}, 1, 0, 1},
    {SS_ISMULH_R, 3, {M_MOV_RR, M_IMUL_R, M_MOV_RR_DEP}, 1, 0, 1},
    {SS_IMUL_RCP, 2, {M_MOV_RI64, M_IMUL_RR_DEP}, 1, 1, -1}};
static const ss_info SS_NOP = {SS_INVALID, 0, {{0, 0, 0, 0, 0}}, 0, 0, 0};

typedef struct { int n, index; int counts[4]; } decode_buffer;
static const decode_buffer DB_484 = {3, 0, {4, 8, 4}}, DB_7333 = {4, 1, {7, 3, 3, 3}}, DB_3733 = {4, 2, {3, 7, 3, 3}},
                           DB_493 = {3, 3, {4, 9, 3}}, DB_4444 = {4, 4, {4, 4, 4, 4}}, DB_3310 = {3, 5, {3, 3, 10}};
static const decode_buffer *const DB_DEFAULTS[4] = {&DB_484, &DB_7333, &DB_3733, &DB_493};

typedef struct { uint8_t data[64]; size_t idx; } b2gen;
static void b2gen_init(b2gen *g, const void *seed, size_t seedlen) {
    memset(g->data, 0, 64);
    memcpy(g->data, seed, seedlen > 60 ? 60 : seedlen);
    store32(g->data + 60, 0);   /* nonce */
    g->idx = 64;
}
static void b2gen_check(b2gen *g, size_t need) {
    if (g->idx + need > 64) { uint8_t t[64]; rxo_blake2b(t, 64, g->data, 64); memcpy(g->data, t, 64); g->idx = 0; }
}
static uint8_t b2gen_byte(b2gen *g) { b2gen_check(g, 1); return g->data[g->idx++]; }
static uint32_t b2gen_u32(b2gen *g) { b2gen_check(g, 4); uint32_t v = load32(g->data + g->idx); g->idx += 4; return v; }

typedef struct { int latency, last_group, last_par; } reg_info;
typedef struct {
    const ss_info *info; int src, dst, mod; uint32_t imm32; int group, group_par, can_reuse, par_is_src;
} ss_instr;

static int is_zero_or_pow2(uint32_t x) { return (x & (x - 1)) == 0; }

static void ss_create(ss_instr *in, const ss_info *info, b2gen *g) {
    in->info = info; in->src = in->dst = -1; in->can_reuse = in->par_is_src = 0; in->mod = 0; in->imm32 = 0; in->group_par = 0;
    switch (info->type) {
        case SS_ISUB_R: in->group = SS_IADD_RS; in->par_is_src = 1; break;
        case SS_IXOR_R: in->group = SS_IXOR_R; in->par_is_src = 1; break;
        case SS_IADD_RS: in->mod = b2gen_byte(g); in->group = SS_IADD_RS; in->par_is_src = 1; break;
        case SS_IMUL_R: in->group = SS_IMUL_R; in->par_is_src = 1; break;
        case SS_IROR_C: do { in->imm32 = b2gen_byte(g) & 63; } while (in->imm32 == 0); in->group = SS_IROR_C; in->group_par = -1; break;
        case SS_IADD_C7: case SS_IADD_C8: case SS_IADD_C9: in->imm32 = b2gen_u32(g); in->group = SS_IADD_C7; in->group_par = -1; break;
        case SS_IXOR_C7: case SS_IXOR_C8: case SS_IXOR_C9: in->imm32 = b2gen_u32(g); in->group = SS_IXOR_C7; in->group_par = -1; break;
        case SS_IMULH_R: in->can_reuse = 1; in->group = SS_IMULH_R; in->group_par = (int)b2gen_u32(g); break;
        case SS_ISMULH_R: in->can_reuse = 1; in->group = SS_ISMULH_R; in->group_par = (int)b2gen_u32(g); break;
        case SS_IMUL_RCP: do { in->imm32 = b2gen_u32(g); } while (is_zero_or_pow2(in->imm32)); in->group = SS_IMUL_RCP; in->group_par = -1; break;
        default: break;
    }
}
static void ss_create_for_slot(ss_instr *in, b2gen *g, int slot, int fetch_type, int is_last) {
    switch (slot) {
        case 3:
            if (is_last) { static const int s3l[4] = {SS_ISUB_R, SS_IXOR_R, SS_IMULH_R, SS_ISMULH_R}; ss_create(in, &SS_INFO[s3l[b2gen_byte(g) & 3]], g); }
            else { static const int s3[2] = {SS_ISUB_R, SS_IXOR_R}; ss_create(in, &SS_INFO[s3[b2gen_byte(g) & 1]], g); }
            break;
        case 4:
            if (fetch_type == 4 && !is_last) ss_create(in, &SS_INFO[SS_IMUL_R], g);
            else { static const int s4[2] = {SS_IROR_C, SS_IADD_RS}; ss_create(in, &SS_INFO[s4[b2gen_byte(g) & 1]], g); }
            break;
        case 7: { static const int s[2] = {SS_IXOR_C7, SS_IADD_C7}; ss_create(in, &SS_INFO[s[b2gen_byte(g) & 1]], g); } break;
        case 8: { static const int s[2] = {SS_IXOR_C8, SS_IADD_C8}; ss_create(in, &SS_INFO[s[b2gen_byte(g) & 1]], g); } break;
        case 9: { static const int s[2] = {SS_IXOR_C9, SS_IADD_C9}; ss_create(in, &SS_INFO[s[b2gen_byte(g) & 1]], g); } break;
        case 10: ss_create(in, &SS_INFO[SS_IMUL_RCP], g); break;
    }
}
static int ss_select_register(const int *avail, int n, b2gen *g, int *reg) {
    if (n == 0) return 0;
    int index = n > 1 ? (int)(b2gen_u32(g) % (uint32_t)n) : 0;
    *reg = avail[index];
    return 1;
}
static int ss_select_dst(ss_instr *in, int cycle, int allow_chained_mul, const reg_info *regs, b2gen *g) {
    int avail[8], n = 0;
    for (int i = 0; i < 8; i++)
        if (regs[i].latency <= cycle && (in->can_reuse || i != in->src) &&
            (allow_chained_mul || in->group != SS_IMUL_R || regs[i].last_group != SS_IMUL_R) &&
            (regs[i].last_group != in->group || regs[i].last_par != in->group_par) &&
            (in->info->type != SS_IADD_RS || i != REG_NEEDS_DISP))
            avail[n++] = i;
    return ss_select_register(avail, n, g, &in->dst);
}
static int ss_select_src(ss_instr *in, int cycle, const reg_info *regs, b2gen *g) {
    int avail[8], n = 0;
    for (int i = 0; i < 8; i++) if (regs[i].latency <= cycle) avail[n++] = i;
    if (n == 2 && in->info->type == SS_IADD_RS && (avail[0] == REG_NEEDS_DISP || avail[1] == REG_NEEDS_DISP)) {
        in->group_par = in->src = REG_NEEDS_DISP;
        return 1;
    }
    if (ss_select_register(avail, n, g, &in->src)) { if (in->par_is_src) in->group_par = in->src; return 1; }
    return 0;
}
static int sched_uop(int uop, int (*busy)[3], int cycle, int commit) {
    for (; cycle < CYCLE_MAP; cycle++) {
        if ((uop & P5) && !busy[cycle][2]) { if (commit) busy[cycle][2] = uop; return cycle; }
        if ((uop & P0) && !busy[cycle][0]) { if (commit) busy[cycle][0] = uop; return cycle; }
        if ((uop & P1) && !busy[cycle][1]) { if (commit) busy[cycle][1] = uop; return cycle; }
    }
    return -1;
}
static int sched_mop(const macro_op *m, int (*busy)[3], int cycle, int dep_cycle, int commit) {
    if (m->uop1 == 0) return cycle;   /* eliminated (register move): takes no port and no dependency wait */
    if (m->dependent && dep_cycle > cycle) cycle = dep_cycle;
    if (m->uop2 == 0) return sched_uop(m->uop1, busy, cycle, commit);
    for (; cycle < CYCLE_MAP; cycle++) {
        int c1 = sched_uop(m->uop1, busy, cycle, 0), c2 = sched_uop(m->uop2, busy, cycle, 0);
        if (c1 >= 0 && c1 == c2) {
            if (commit) { sched_uop(m->uop1, busy, c1, 1); sched_uop(m->uop2, busy, c2, 1); }
            return c1;
        }
    }
    return -1;
}

static void ss_generate(rxo_ss_program *prog, b2gen *g) {
    int busy[CYCLE_MAP][3];
    memset(busy, 0, sizeof busy);
    reg_info regs[8];
    for (int i = 0; i < 8; i++) { regs[i].latency = 0; regs[i].last_group = SS_INVALID; regs[i].last_par = -1; }
    const decode_buffer *db = NULL;
    ss_instr cur; memset(&cur, 0, sizeof cur); cur.info = &SS_NOP; cur.src = cur.dst = -1;
    int mop_index = 0, cycle = 0, dep_cycle = 0, retire_cycle = 0, saturated = 0, prog_size = 0, mul_count = 0, throw_away = 0;
    (void)retire_cycle;
    for (int decode_cycle = 0; decode_cycle < SS_LATENCY && !saturated && prog_size < SS_MAXSIZE; decode_cycle++) {
        /* fetch configuration for this decode cycle (16 bytes of x86 code) */
        int t = cur.info->type;
        if (t == SS_IMULH_R || t == SS_ISMULH_R) db = &DB_3310;
        else if (mul_count < decode_cycle + 1) db = &DB_4444;
        else if (t == SS_IMUL_RCP) db = (b2gen_byte(g) & 1) ? &DB_484 : &DB_493;
        else db = DB_DEFAULTS[b2gen_byte(g) & 3];
        int bi = 0;
        while (bi < db->n) {
            int top_cycle = cycle;
            if (mop_index >= cur.info->nops) {
                if (saturated || prog_size >= SS_MAXSIZE) break;
                ss_create_for_slot(&cur, g, db->counts[bi], db->index, db->n == bi + 1);
                mop_index = 0;
            }
            const macro_op *mop = &cur.info->ops[mop_index];
            int sc = sched_mop(mop, busy, cycle, dep_cycle, 0);
            if (sc < 0) { saturated = 1; break; }
            if (mop_index == cur.info->src_op) {
                int fwd;
                for (fwd = 0; fwd < LOOK_FORWARD && !ss_select_src(&cur, sc, regs, g); fwd++) { sc++; cycle++; }
                if (fwd == LOOK_FORWARD) {
                    if (throw_away < MAX_THROWAWAY) { throw_away++; mop_index = cur.info->nops; continue; }
                    cur.info = &SS_NOP; break;
                }
            }
            if (mop_index == cur.info->dst_op) {
                int fwd;
                for (fwd = 0; fwd < LOOK_FORWARD && !ss_select_dst(&cur, sc, throw_away > 0, regs, g); fwd++) { sc++; cycle++; }
                if (fwd == LOOK_FORWARD) {
                    if (throw_away < MAX_THROWAWAY) { throw_away++; mop_index = cur.info->nops; continue; }
                    cur.info = &SS_NOP; break;
                }
            }
            throw_away = 0;
            sc = sched_mop(mop, busy, sc, sc, 1);
            if (sc < 0) { saturated = 1; break; }
            dep_cycle = sc + mop->latency;
            if (mop_index == cur.info->result_op) {
                reg_info *ri = &regs[cur.dst];
                retire_cycle = dep_cycle;
                ri->latency = retire_cycle; ri->last_group = cur.group; ri->last_par = cur.group_par;
            }
            bi++; mop_index++;
            if (sc >= SS_LATENCY) saturated = 1;
            cycle = top_cycle;
            if (mop_index >= cur.info->nops) {
                rxo_ss_instr *o = &prog->ins[prog_size++];
                o->opcode = (uint8_t)cur.info->type; o->dst = (uint8_t)cur.dst; o->src = (uint8_t)(cur.src >= 0 ? cur.src : cur.dst);
                o->mod = (uint8_t)cur.mod; o->imm32 = cur.imm32;
                mul_count += (cur.info->type == SS_IMUL_R || cur.info->type == SS_IMULH_R || cur.info->type == SS_ISMULH_R || cur.info->type == SS_IMUL_RCP);
            }
        }
        cycle++;
    }
    /* address register = the one with the highest latency on an idealised unlimited-width machine */
    int asic[8] = {0};
    for (int i = 0; i < prog_size; i++) {
        const rxo_ss_instr *o = &prog->ins[i];
        int ld = asic[o->dst] + 1, ls = o->dst != o->src ? asic[o->src] + 1 : 0;
        asic[o->dst] = ld > ls ? ld : ls;
    }
    int best = 0, addr = 0;
    for (int i = 0; i < 8; i++) if (asic[i] > best) { best = asic[i]; addr = i; }
    prog->size = (uint32_t)prog_size;
    prog->address_reg = (uint32_t)addr;
}

uint64_t rxo_reciprocal(uint32_t divisor) {
    const uint64_t p2exp63 = 1ULL << 63;
    uint64_t quotient = p2exp63 / divisor, remainder = p2exp63 % divisor;
    unsigned bsr = 0;
    for (uint32_t bit = divisor; bit > 0; bit >>= 1) bsr++;
    for (unsigned shift = 0; shift < bsr; shift++) {
        if (remainder >= divisor - remainder) { quotient = quotient * 2 + 1; remainder = remainder * 2 - divisor; }
        else { quotient = quotient * 2; remainder = remainder * 2; }
    }
    return quotient;
}
static inline uint64_t mulh(uint64_t a, uint64_t b) { return (uint64_t)(((unsigned __int128)a * b) >> 64); }
static inline int64_t smulh(int64_t a, int64_t b) { return (int64_t)(((__int128)a * b) >> 64); }
static inline uint64_t sext32(uint32_t x) { return (uint64_t)(int64_t)(int32_t)x; }

static void ss_execute(uint64_t r[8], const rxo_ss_program *p) {
    for (uint32_t j = 0; j < p->size; j++) {
        const rxo_ss_instr *o = &p->ins[j];
        switch (o->opcode) {
            case SS_ISUB_R: r[o->dst] -= r[o->src]; break;
            case SS_IXOR_R: r[o->dst] ^= r[o->src]; break;
            case SS_IADD_RS: r[o->dst] += r[o->src] << ((o->mod >> 2) & 3); break;
            case SS_IMUL_R: r[o->dst] *= r[o->src]; break;
            case SS_IROR_C: r[o->dst] = rotr64(r[o->dst], o->imm32 & 63); break;
            case SS_IADD_C7: case SS_IADD_C8: case SS_IADD_C9: r[o->dst] += sext32(o->imm32); break;
            case SS_IXOR_C7: case SS_IXOR_C8: case SS_IXOR_C9: r[o->dst] ^= sext32(o->imm32); break;
            case SS_IMULH_R: r[o->dst] = mulh(r[o->dst], r[o->src]); break;
            case SS_ISMULH_R: r[o->dst] = (uint64_t)smulh((int64_t)r[o->dst], (int64_t)r[o->src]); break;
            case SS_IMUL_RCP: r[o->dst] *= o->rcp; break;
        }
    }
}

/* ------------------------------------------------------------------------------------------------ */
/* Cache, dataset items (spec §7)                                                                     */
/* ------------------------------------------------------------------------------------------------ */
#define RX_ARGON_MEMORY 262144u
#define RX_ARGON_ITERS 3u
#define RX_CACHE_ACCESSES 8
#define RX_DATASET_BASE (2147483648ULL)
#define RX_DATASET_EXTRA (33554368ULL)
#define RX_DATASET_ITEMS ((RX_DATASET_BASE + RX_DATASET_EXTRA) / 64)
#define RX_SCRATCHPAD_L3 2097152u
#define RX_SCRATCHPAD_L2 262144u
#define RX_SCRATCHPAD_L1 16384u
#define RX_PROGRAM_SIZE 256
#define RX_PROGRAM_ITERS 2048
#define RX_PROGRAM_COUNT 8

struct rxo_cache {
    uint64_t *memory;            /* 256 MiB */
    rxo_ss_program programs[RX_CACHE_ACCESSES];
    uint8_t *dataset;            /* optional 2080 MiB (fast mode) */
};

rxo_cache *rxo_cache_new(const void *key, size_t keylen) {
    rx_consts();
    rxo_cache *c = (rxo_cache *)calloc(1, sizeof *c);
    if (!c) return NULL;
    if (posix_memalign((void **)&c->memory, 64, (size_t)RX_ARGON_MEMORY * 1024)) { free(c); return NULL; }
    rxo_argon2d_fill(c->memory, RX_ARGON_MEMORY, RX_ARGON_ITERS, key, (uint32_t)keylen, "RandomX\x03", 8, 0, NULL);
    b2gen g; b2gen_init(&g, key, keylen);
    for (int i = 0; i < RX_CACHE_ACCESSES; i++) {
        ss_generate(&c->programs[i], &g);
        for (uint32_t j = 0; j < c->programs[i].size; j++)
            if (c->programs[i].ins[j].opcode == SS_IMUL_RCP) c->programs[i].ins[j].rcp = rxo_reciprocal(c->programs[i].ins[j].imm32);
    }
    return c;
}
void rxo_cache_free(rxo_cache *c) { if (c) { free(c->memory); free(c->dataset); free(c); } }
const uint64_t *rxo_cache_memory(const rxo_cache *c) { return c->memory; }
const rxo_ss_program *rxo_cache_programs(const rxo_cache *c) { return c->programs; }

void rxo_dataset_item(const rxo_cache *c, uint64_t item, uint64_t out[8]) {
    static const uint64_t MUL0 = 6364136223846793005ULL;
    static const uint64_t ADD[8] = {0, 9298411001130361340ULL, 12065312585734608966ULL, 9306329213124626780ULL,
                                    5281919268842080866ULL, 10536153434571861004ULL, 3398623926847679864ULL, 9549104520008361294ULL};
    uint64_t r[8], reg = item;
    r[0] = (item + 1) * MUL0;
    for (int i = 1; i < 8; i++) r[i] = r[0] ^ ADD[i];
    const uint64_t mask = ((size_t)RX_ARGON_MEMORY * 1024) / 64 - 1;
    for (int i = 0; i < RX_CACHE_ACCESSES; i++) {
        const uint64_t *mix = c->memory + (reg & mask) * 8;
        ss_execute(r, &c->programs[i]);
        for (int q = 0; q < 8; q++) r[q] ^= mix[q];
        reg = r[c->programs[i].address_reg];
    }
    memcpy(out, r, 64);
}

typedef struct { rxo_cache *c; uint64_t lo, hi; } ds_job;
static void *ds_worker(void *a) {
    ds_job *j = (ds_job *)a;
    for (uint64_t i = j->lo; i < j->hi; i++) rxo_dataset_item(j->c, i, (uint64_t *)(j->c->dataset + i * 64));
    return NULL;
}
int rxo_dataset_init(rxo_cache *c, int threads) {
    if (c->dataset) return 0;
    if (posix_memalign((void **)&c->dataset, 64, RX_DATASET_ITEMS * 64)) { c->dataset = NULL; return -1; }
    if (threads < 1) threads = 1;
    pthread_t th[256]; ds_job jobs[256];
    if (threads > 256) threads = 256;
    uint64_t per = (RX_DATASET_ITEMS + threads - 1) / threads;
    for (int t = 0; t < threads; t++) {
        jobs[t].c = c; jobs[t].lo = per * t; jobs[t].hi = per * (t + 1) > RX_DATASET_ITEMS ? RX_DATASET_ITEMS : per * (t + 1);
        if (jobs[t].lo > jobs[t].hi) jobs[t].lo = jobs[t].hi;
        pthread_create(&th[t], NULL, ds_worker, &jobs[t]);
    }
    for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
    return 0;
}
int rxo_has_dataset(const rxo_cache *c) { return c->dataset != NULL; }
const uint8_t *rxo_dataset_memory(const rxo_cache *c) { return c->dataset; }

/* ------------------------------------------------------------------------------------------------ */
/* The virtual machine (spec §4, §5)                                                                  */
/* ------------------------------------------------------------------------------------------------ */
enum { I_IADD_RS, I_IADD_M, I_ISUB_R, I_ISUB_M, I_IMUL_R, I_IMUL_M, I_IMULH_R, I_IMULH_M, I_ISMULH_R, I_ISMULH_M, I_IMUL_RCP,
       I_INEG_R, I_IXOR_R, I_IXOR_M, I_IROR_R, I_IROL_R, I_ISWAP_R, I_FSWAP_R, I_FADD_R, I_FADD_M, I_FSUB_R, I_FSUB_M,
       I_FSCAL_R, I_FMUL_R, I_FDIV_M, I_FSQRT_R, I_CBRANCH, I_CFROUND, I_ISTORE, I_NOP, I_COUNT };
/* instruction frequencies out of 256 (spec table 5.1), in opcode order */
static const uint8_t FREQ[I_COUNT] = {16, 7, 16, 7, 16, 4, 4, 1, 4, 1, 8, 2, 15, 5, 8, 2, 4, 4, 16, 5, 16, 5, 6, 32, 4, 6, 25, 1, 16, 0};
static uint8_t OPMAP[256];
static int g_opmap_ready;
static void opmap_init(void) {
    if (g_opmap_ready) return;
    int k = 0;
    for (int t = 0; t < I_COUNT; t++) for (int j = 0; j < FREQ[t]; j++) OPMAP[k++] = (uint8_t)t;
    __sync_synchronize();
    g_opmap_ready = 1;
}
void rxo_opcode_map(uint8_t out[256]) { opmap_init(); memcpy(out, OPMAP, 256); }

#define L1_MASK ((RX_SCRATCHPAD_L1 - 1) & ~7u)
#define L2_MASK ((RX_SCRATCHPAD_L2 - 1) & ~7u)
#define L3_MASK ((RX_SCRATCHPAD_L3 - 1) & ~7u)
#define L3_MASK64 ((RX_SCRATCHPAD_L3 - 1) & ~63u)
#define CACHELINE_ALIGN_MASK ((uint32_t)((RX_DATASET_BASE - 1) & ~63ULL))
#define DATASET_EXTRA_ITEMS (RX_DATASET_EXTRA / 64)

typedef struct {
    uint8_t type, dst, src, pad;
    uint32_t mem_mask;
    uint64_t imm;
    int32_t target;
    uint32_t shift;
} dec_instr;

typedef struct {
    uint64_t r[8];
    __m128d f[4], e[4], a[4];
} vm_regs;

static void vm_decode(const uint8_t *prog /* 256 x 8 bytes */, dec_instr *out) {
    int usage[8];
    for (int i = 0; i < 8; i++) usage[i] = -1;
    for (int i = 0; i < RX_PROGRAM_SIZE; i++) {
        const uint8_t *p = prog + 8 * i;
        uint8_t opcode = p[0], dstb = p[1], srcb = p[2], mod = p[3];
        uint32_t imm32 = load32(p + 4);
        dec_instr *d = &out[i];
        memset(d, 0, sizeof *d);
        int t = OPMAP[opcode];
        int dst = dstb & 7, src = srcb & 7;
        d->type = (uint8_t)t; d->dst = (uint8_t)dst; d->src = (uint8_t)src;
        switch (t) {
            case I_IADD_RS:
                d->shift = (mod >> 2) & 3;
                d->imm = dst == REG_NEEDS_DISP ? sext32(imm32) : 0;
                usage[dst] = i; break;
            case I_IADD_M: case I_ISUB_M: case I_IMUL_M: case I_IMULH_M: case I_ISMULH_M: case I_IXOR_M:
                d->imm = sext32(imm32);
                if (src != dst) d->mem_mask = (mod & 3) ? L1_MASK : L2_MASK;
                else { d->src = 8; d->mem_mask = L3_MASK; }     /* src 8 = constant zero */
                usage[dst] = i; break;
            case I_ISUB_R: case I_IMUL_R: case I_IXOR_R:
                if (src == dst) { d->src = 9; d->imm = sext32(imm32); }   /* src 9 = immediate */
                usage[dst] = i; break;
            case I_IMULH_R: case I_ISMULH_R: usage[dst] = i; break;
            case I_IMUL_RCP:
                if (!is_zero_or_pow2(imm32)) { d->type = I_IMUL_R; d->src = 9; d->imm = rxo_reciprocal(imm32); usage[dst] = i; }
                else d->type = I_NOP;
                break;
            case I_INEG_R: usage[dst] = i; break;
            case I_IROR_R: case I_IROL_R:
                if (src == dst) { d->src = 9; d->imm = imm32; }
                usage[dst] = i; break;
            case I_ISWAP_R:
                if (src != dst) { usage[dst] = i; usage[src] = i; } else d->type = I_NOP;
                break;
            case I_FSWAP_R: break;   /* dst 0-3 = f, 4-7 = e */
            case I_FADD_R: case I_FSUB_R: case I_FMUL_R: d->dst = dstb & 3; d->src = srcb & 3; break;
            case I_FADD_M: case I_FSUB_M: case I_FDIV_M:
                d->dst = dstb & 3; d->mem_mask = (mod & 3) ? L1_MASK : L2_MASK; d->imm = sext32(imm32); break;
            case I_FSCAL_R: case I_FSQRT_R: d->dst = dstb & 3; break;
            case I_CBRANCH: {
                d->target = usage[dst];
                int shift = (mod >> 4) + 8;
                d->imm = (sext32(imm32) | (1ULL << shift)) & ~(1ULL << (shift - 1));
                d->mem_mask = 0; d->shift = (uint32_t)shift;
                for (int j = 0; j < 8; j++) usage[j] = i;
            } break;
            case I_CFROUND: d->imm = imm32 & 63; break;
            case I_ISTORE:
                d->imm = sext32(imm32);
                d->mem_mask = (mod >> 4) < 14 ? ((mod & 3) ? L1_MASK : L2_MASK) : L3_MASK;
                break;
            default: break;
        }
    }
}

static inline __m128d cvt_i32x2(const uint8_t *p) { return _mm_cvtepi32_pd(_mm_loadl_epi64((const __m128i *)p)); }
static inline void set_rounding(uint32_t mode) { _mm_setcsr(0x9FC0u | (mode << 13)); }

typedef struct {
    uint8_t *scratchpad;   /* 2 MiB */
    vm_regs reg;
    uint64_t emask[2];
    uint32_t ma, mx, read_reg[4];
    uint64_t dataset_offset;
    dec_instr code[RX_PROGRAM_SIZE];
    uint8_t program[128 + 8 * RX_PROGRAM_SIZE];
} vm_t;

static inline __m128d mask_e(const vm_t *vm, __m128d x) {
    const __m128i mant = _mm_set1_epi64x((long long)((1ULL << 56) - 1));
    const __m128i em = _mm_set_epi64x((long long)vm->emask[1], (long long)vm->emask[0]);
    return _mm_castsi128_pd(_mm_or_si128(_mm_and_si128(_mm_castpd_si128(x), mant), em));
}
static uint64_t small_positive_float_bits(uint64_t entropy) {
    uint64_t exponent = entropy >> 59, mantissa = entropy & ((1ULL << 52) - 1);
    exponent += 1023; exponent &= 2047; exponent <<= 52;
    return exponent | mantissa;
}
static uint64_t float_mask(uint64_t entropy) {
    uint64_t exponent = 0x300;
    exponent |= (entropy >> 60) << 4;
    exponent <<= 52;
    return (entropy & ((1ULL << 22) - 1)) | exponent;
}

static void vm_run(vm_t *vm, const rxo_cache *cache, const uint8_t seed[64]) {
    rxo_fill_aes_4rx4(seed, sizeof vm->program, vm->program);
    uint64_t ent[16];
    memcpy(ent, vm->program, 128);
    vm_decode(vm->program + 128, vm->code);
    vm_regs *R = &vm->reg;
    for (int i = 0; i < 4; i++) {
        uint64_t lo = small_positive_float_bits(ent[2 * i]), hi = small_positive_float_bits(ent[2 * i + 1]);
        R->a[i] = _mm_castsi128_pd(_mm_set_epi64x((long long)hi, (long long)lo));
    }
    vm->ma = (uint32_t)ent[8] & CACHELINE_ALIGN_MASK;
    vm->mx = (uint32_t)ent[10];
    uint64_t ar = ent[12];
    for (int i = 0; i < 4; i++) { vm->read_reg[i] = 2 * i + (ar & 1); ar >>= 1; }
    vm->dataset_offset = (ent[13] % (DATASET_EXTRA_ITEMS + 1)) * 64;
    vm->emask[0] = float_mask(ent[14]); vm->emask[1] = float_mask(ent[15]);
    for (int i = 0; i < 8; i++) R->r[i] = 0;

    uint8_t *sp = vm->scratchpad;
    uint32_t sp0 = vm->mx, sp1 = vm->ma;
    const __m128d scal = _mm_castsi128_pd(_mm_set1_epi64x((long long)0x80F0000000000000ULL));
    for (int ic = 0; ic < RX_PROGRAM_ITERS; ic++) {
        uint64_t mix = R->r[vm->read_reg[0]] ^ R->r[vm->read_reg[1]];
        sp0 ^= (uint32_t)mix; sp0 &= L3_MASK64;
        sp1 ^= (uint32_t)(mix >> 32); sp1 &= L3_MASK64;
        for (int i = 0; i < 8; i++) R->r[i] ^= load64(sp + sp0 + 8 * i);
        for (int i = 0; i < 4; i++) R->f[i] = cvt_i32x2(sp + sp1 + 8 * i);
        for (int i = 0; i < 4; i++) R->e[i] = mask_e(vm, cvt_i32x2(sp + sp1 + 8 * (4 + i)));

        for (int pc = 0; pc < RX_PROGRAM_SIZE; pc++) {
            const dec_instr *d = &vm->code[pc];
            uint64_t srcv = d->src < 8 ? R->r[d->src] : (d->src == 8 ? 0 : d->imm);
            switch (d->type) {
                case I_IADD_RS: R->r[d->dst] += (R->r[d->src] << d->shift) + d->imm; break;
                case I_IADD_M: R->r[d->dst] += load64(sp + ((srcv + d->imm) & d->mem_mask)); break;
                case I_ISUB_R: R->r[d->dst] -= srcv; break;
                case I_ISUB_M: R->r[d->dst] -= load64(sp + ((srcv + d->imm) & d->mem_mask)); break;
                case I_IMUL_R: R->r[d->dst] *= srcv; break;
                case I_IMUL_M: R->r[d->dst] *= load64(sp + ((srcv + d->imm) & d->mem_mask)); break;
                case I_IMULH_R: R->r[d->dst] = mulh(R->r[d->dst], R->r[d->src]); break;
                case I_IMULH_M: R->r[d->dst] = mulh(R->r[d->dst], load64(sp + ((srcv + d->imm) & d->mem_mask))); break;
                case I_ISMULH_R: R->r[d->dst] = (uint64_t)smulh((int64_t)R->r[d->dst], (int64_t)R->r[d->src]); break;
                case I_ISMULH_M: R->r[d->dst] = (uint64_t)smulh((int64_t)R->r[d->dst], (int64_t)load64(sp + ((srcv + d->imm) & d->mem_mask))); break;
                case I_INEG_R: R->r[d->dst] = ~R->r[d->dst] + 1; break;
                case I_IXOR_R: R->r[d->dst] ^= srcv; break;
                case I_IXOR_M: R->r[d->dst] ^= load64(sp + ((srcv + d->imm) & d->mem_mask)); break;
                case I_IROR_R: R->r[d->dst] = rotr64(R->r[d->dst], (unsigned)(srcv & 63)); break;
                case I_IROL_R: R->r[d->dst] = rotl64(R->r[d->dst], (unsigned)(srcv & 63)); break;
                case I_ISWAP_R: { uint64_t t = R->r[d->dst]; R->r[d->dst] = R->r[d->src]; R->r[d->src] = t; } break;
                case I_FSWAP_R: {
                    __m128d *x = d->dst < 4 ? &R->f[d->dst] : &R->e[d->dst - 4];
                    *x = _mm_shuffle_pd(*x, *x, 1);
                } break;
                case I_FADD_R: R->f[d->dst] = _mm_add_pd(R->f[d->dst], R->a[d->src]); break;
                case I_FADD_M: R->f[d->dst] = _mm_add_pd(R->f[d->dst], cvt_i32x2(sp + ((R->r[d->src] + d->imm) & d->mem_mask))); break;
                case I_FSUB_R: R->f[d->dst] = _mm_sub_pd(R->f[d->dst], R->a[d->src]); break;
                case I_FSUB_M: R->f[d->dst] = _mm_sub_pd(R->f[d->dst], cvt_i32x2(sp + ((R->r[d->src] + d->imm) & d->mem_mask))); break;
                case I_FSCAL_R: R->f[d->dst] = _mm_xor_pd(R->f[d->dst], scal); break;
                case I_FMUL_R: R->e[d->dst] = _mm_mul_pd(R->e[d->dst], R->a[d->src]); break;
                case I_FDIV_M: R->e[d->dst] = _mm_div_pd(R->e[d->dst], mask_e(vm, cvt_i32x2(sp + ((R->r[d->src] + d->imm) & d->mem_mask)))); break;
                case I_FSQRT_R: R->e[d->dst] = _mm_sqrt_pd(R->e[d->dst]); break;
                case I_CBRANCH:
                    R->r[d->dst] += d->imm;
                    if ((R->r[d->dst] & (255ULL << d->shift)) == 0) pc = d->target;
                    break;
                case I_CFROUND: set_rounding((uint32_t)(rotr64(R->r[d->src], (unsigned)d->imm) & 3)); break;
                case I_ISTORE: store64(sp + ((R->r[d->dst] + d->imm) & d->mem_mask), R->r[d->src]); break;
                default: break;
            }
        }

        vm->mx ^= (uint32_t)(R->r[vm->read_reg[2]] ^ R->r[vm->read_reg[3]]);
        vm->mx &= CACHELINE_ALIGN_MASK;
        {
            uint64_t addr = vm->dataset_offset + vm->ma, item[8];
            const uint64_t *line;
            if (cache->dataset) line = (const uint64_t *)(cache->dataset + addr);
            else { rxo_dataset_item(cache, addr / 64, item); line = item; }
            for (int i = 0; i < 8; i++) R->r[i] ^= line[i];
        }
        { uint32_t t = vm->mx; vm->mx = vm->ma; vm->ma = t; }
        for (int i = 0; i < 8; i++) store64(sp + sp1 + 8 * i, R->r[i]);
        for (int i = 0; i < 4; i++) R->f[i] = _mm_xor_pd(R->f[i], R->e[i]);
        for (int i = 0; i < 4; i++) _mm_storeu_pd((double *)(sp + sp0 + 16 * i), R->f[i]);
        sp0 = 0; sp1 = 0;
    }
}

static void vm_regfile_bytes(const vm_t *vm, uint8_t out[256]) {
    memcpy(out, vm->reg.r, 64);
    for (int i = 0; i < 4; i++) {
        _mm_storeu_pd((double *)(out + 64 + 16 * i), vm->reg.f[i]);
        _mm_storeu_pd((double *)(out + 128 + 16 * i), vm->reg.e[i]);
        _mm_storeu_pd((double *)(out + 192 + 16 * i), vm->reg.a[i]);
    }
}

struct rxo_vm { vm_t vm; };
rxo_vm *rxo_vm_new(void) {
    opmap_init(); rx_consts();
    rxo_vm *v = NULL;
    if (posix_memalign((void **)&v, 64, sizeof *v)) return NULL;
    memset(v, 0, sizeof *v);
    if (posix_memalign((void **)&v->vm.scratchpad, 64, RX_SCRATCHPAD_L3)) { free(v); return NULL; }
    return v;
}
void rxo_vm_free(rxo_vm *v) { if (v) { free(v->vm.scratchpad); free(v); } }

/* randomx_calculate_hash (spec §2): Blake2b seed -> scratchpad -> 8 chained programs -> AesHash1R -> Blake2b-256.
 * trace (optional, 8 x 256 bytes): the register file after each program (tests compare the GPU against it). */
void rxo_hash_vm(rxo_vm *v, const rxo_cache *cache, const void *input, size_t inlen, uint8_t out[32], uint8_t *trace) {
    unsigned saved_csr = _mm_getcsr();
    uint8_t seed[64], rf[256];
    vm_t *vm = &v->vm;
    rxo_blake2b(seed, 64, input, inlen);
    rxo_fill_aes_1rx4(seed, RX_SCRATCHPAD_L3, vm->scratchpad);
    set_rounding(0);
    for (int chain = 0; chain < RX_PROGRAM_COUNT; chain++) {
        vm_run(vm, cache, seed);
        vm_regfile_bytes(vm, rf);
        if (trace) memcpy(trace + 256 * chain, rf, 256);
        if (chain < RX_PROGRAM_COUNT - 1) rxo_blake2b(seed, 64, rf, 256);
    }
    rxo_hash_aes_1rx4(vm->scratchpad, RX_SCRATCHPAD_L3, rf + 192);
    rxo_blake2b(out, 32, rf, 256);
    _mm_setcsr(saved_csr);
}
void rxo_hash(const rxo_cache *cache, const void *input, size_t inlen, uint8_t out[32]) {
    rxo_vm *v = rxo_vm_new();
    rxo_hash_vm(v, cache, input, inlen, out, NULL);
    rxo_vm_free(v);
}

/* ------------------------------------------------------------------------------------------------ */
/* k2pow on top of it (post-rs pow/randomx.rs, recollection — see PARITY STATUS)                      */
/* ------------------------------------------------------------------------------------------------ */
void rxo_k2pow_input(uint64_t pow, uint8_t nonce_group, const uint8_t challenge8[8], const uint8_t node_id[32], uint8_t out[48]) {
    for (int i = 0; i < 7; i++) out[i] = (uint8_t)(pow >> (8 * i));
    out[7] = nonce_group;
    memcpy(out + 8, challenge8, 8);
    memcpy(out + 16, node_id, 32);
}
typedef struct {
    const rxo_cache *cache; uint8_t nonce_group; const uint8_t *challenge8, *node_id, *difficulty;
    uint64_t start, count; int tid, nthreads; uint8_t *hashes; volatile uint64_t *best; volatile int *stop; int stop_at_first;
} k2_job;
static void *k2_worker(void *a) {
    k2_job *j = (k2_job *)a;
    rxo_vm *v = rxo_vm_new();
    uint8_t in[48], h[32];
    for (uint64_t i = (uint64_t)j->tid; i < j->count; i += (uint64_t)j->nthreads) {
        if (j->stop_at_first && *j->stop) break;
        uint64_t pow = j->start + i;
        rxo_k2pow_input(pow, j->nonce_group, j->challenge8, j->node_id, in);
        rxo_hash_vm(v, j->cache, in, 48, h, NULL);
        if (j->hashes) memcpy(j->hashes + 32 * i, h, 32);
        if (j->difficulty && memcmp(h, j->difficulty, 32) < 0) {
            uint64_t cur;
            do { cur = *j->best; if (pow >= cur) break; } while (!__sync_bool_compare_and_swap(j->best, cur, pow));
            if (j->stop_at_first) *j->stop = 1;
        }
    }
    rxo_vm_free(v);
    return NULL;
}
/* Hashes pow = start .. start+count-1; hashes (optional) receives count x 32 bytes; *found_pow = the smallest pow in the
 * range whose hash is < difficulty (big-endian byte compare), or UINT64_MAX.  Returns elapsed seconds. */
double rxo_k2pow_scan(const rxo_cache *cache, uint8_t nonce_group, const uint8_t challenge8[8], const uint8_t node_id[32],
                      const uint8_t *difficulty, uint64_t start, uint64_t count, int threads, uint8_t *hashes, uint64_t *found_pow) {
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    pthread_t th[256]; k2_job jobs[256];
    volatile uint64_t best = UINT64_MAX; volatile int stop = 0;
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int t = 0; t < threads; t++) {
        jobs[t] = (k2_job){cache, nonce_group, challenge8, node_id, difficulty, start, count, t, threads, hashes, &best, &stop, 0};
        pthread_create(&th[t], NULL, k2_worker, &jobs[t]);
    }
    for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    if (found_pow) *found_pow = best;
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
