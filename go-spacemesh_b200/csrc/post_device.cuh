// post_device.cuh — per-thread arithmetic of the POST label function for sm_90a.
//
// label32(i) = scrypt_jane(P = commitment[32] || LE64(i) || 0^32, S = "", N, r = 1, p = 1, dkLen = 32)
// where scrypt_jane is scrypt's structure (PBKDF2 -> ROMix -> PBKDF2, RFC 7914 §6) with ChaCha20/8 as the
// BlockMix core and HMAC-Keccak-512 (original 0x01 padding, 72-byte block) inside PBKDF2 — floodyberry's
// scrypt-jane as libpost builds it.  This is the function go-spacemesh reaches through activation/post.go:295
// `mgr.init.Initialize` and activation/post_verifier.go:159 `ProofVerifier.Verify`; it is pinned against the real
// VRF nonces of the reference's checkpoint fixture (tests/golden/checkpoint_vrf.json).
//
// Everything here is HD (host+device) so that tests/host_emul.cpp can run the exact same
// per-thread code on the CPU against the oracle before any GPU time is spent.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define PD_HD __host__ __device__ __forceinline__
#define PD_D __device__ __forceinline__
#else
#define PD_HD inline
#define PD_D inline
#endif

namespace b200post {

// ------------------------------------------------------------------------------------------------
// rotates.  On the device `rotl` is one SHF.L.W; the byte-aligned ChaCha rotates (16, 8) can also be one PRMT.
// Both issue on the alu pipe (DESIGN.md §K2); ROT selects the form so that the sweep can compare them.
// ------------------------------------------------------------------------------------------------
PD_HD uint32_t rotl(uint32_t x, int k) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(x, x, k);
#else
    return (x << k) | (x >> (32 - k));
#endif
}
PD_HD uint32_t bswap32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __byte_perm(x, 0, 0x0123);
#else
    return (x >> 24) | ((x >> 8) & 0xff00u) | ((x << 8) & 0xff0000u) | (x << 24);
#endif
}
template <int ROT>
PD_HD uint32_t rotl16(uint32_t x) {
#if defined(__CUDA_ARCH__)
    if (ROT & 1) return __byte_perm(x, 0, 0x1032);
#endif
    return rotl(x, 16);
}
template <int ROT>
PD_HD uint32_t rotl8(uint32_t x) {
#if defined(__CUDA_ARCH__)
    if (ROT & 1) return __byte_perm(x, 0, 0x2103);
#endif
    return rotl(x, 8);
}

// ------------------------------------------------------------------------------------------------
// ChaCha20/8 core as scrypt-jane uses it (chacha_core_basic): the 64-byte block is the whole state, four
// double rounds (columns, diagonals), x <- x + rounds(x).  Per quarter-round step: one add (fma/alu pipes), one
// XOR and one rotate (alu pipe) — 256 alu-pipe instructions per core, the kernel's bound (DESIGN.md §5).
// ROT bit 0: 16- and 8-bit rotates as PRMT instead of SHF.
// ------------------------------------------------------------------------------------------------
#define PD_QR(w, a, b, c, d)                                          \
    w[a] += w[b]; w[d] = rotl16<ROT>(w[d] ^ w[a]);                    \
    w[c] += w[d]; w[b] = rotl(w[b] ^ w[c], 12);                       \
    w[a] += w[b]; w[d] = rotl8<ROT>(w[d] ^ w[a]);                     \
    w[c] += w[d]; w[b] = rotl(w[b] ^ w[c], 7);
#define PD_DOUBLE_ROUND(w)                                                                \
    PD_QR(w, 0, 4, 8, 12) PD_QR(w, 1, 5, 9, 13) PD_QR(w, 2, 6, 10, 14) PD_QR(w, 3, 7, 11, 15) \
    PD_QR(w, 0, 5, 10, 15) PD_QR(w, 1, 6, 11, 12) PD_QR(w, 2, 7, 8, 13) PD_QR(w, 3, 4, 9, 14)

template <int ROT, int DR_UNROLL = 4>
PD_HD void chacha20_8(uint32_t (&x)[16]) {
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = x[i];
#pragma unroll DR_UNROLL
    for (int r = 0; r < 4; r++) { PD_DOUBLE_ROUND(w) }
#pragma unroll
    for (int i = 0; i < 16; i++) x[i] += w[i];
}

// Two independent cores in one instruction stream (8 independent dependency chains): used by
// the pipelined ROMix kernel, where every thread advances a filling and a mixing label together.
template <int ROT, int DR_UNROLL>
PD_HD void chacha20_8_x2(uint32_t (&xa)[16], uint32_t (&xb)[16]) {
    uint32_t wa[16], wb[16];
#pragma unroll
    for (int i = 0; i < 16; i++) { wa[i] = xa[i]; wb[i] = xb[i]; }
#pragma unroll DR_UNROLL
    for (int r = 0; r < 4; r++) { PD_DOUBLE_ROUND(wa) PD_DOUBLE_ROUND(wb) }
#pragma unroll
    for (int i = 0; i < 16; i++) { xa[i] += wa[i]; xb[i] += wb[i]; }
}

// scrypt BlockMix for r = 1 (RFC 7914 §4 with the ChaCha core) on X = lo(16) || hi(16):
//   T = hi ^ lo; Y0 = Core(T); Y1 = Core(Y0 ^ hi); X = Y0 || Y1.
template <int ROT, int DR_UNROLL = 4>
PD_HD void blockmix_r1(uint32_t (&lo)[16], uint32_t (&hi)[16]) {
#pragma unroll
    for (int i = 0; i < 16; i++) lo[i] ^= hi[i];
    chacha20_8<ROT, DR_UNROLL>(lo);
#pragma unroll
    for (int i = 0; i < 16; i++) hi[i] ^= lo[i];
    chacha20_8<ROT, DR_UNROLL>(hi);
}
// Same, fused with the ROMix phase-2 "X ^= V[j]" so that the three-way XOR is one LOP3 per word.
template <int ROT, int DR_UNROLL = 4>
PD_HD void blockmix_r1_xor(uint32_t (&lo)[16], uint32_t (&hi)[16], const uint32_t (&vlo)[16],
                           const uint32_t (&vhi)[16]) {
#pragma unroll
    for (int i = 0; i < 16; i++) { hi[i] ^= vhi[i]; lo[i] = lo[i] ^ vlo[i] ^ hi[i]; }
    chacha20_8<ROT, DR_UNROLL>(lo);
#pragma unroll
    for (int i = 0; i < 16; i++) hi[i] ^= lo[i];
    chacha20_8<ROT, DR_UNROLL>(hi);
}

// One ROMix step of a dual-label kernel: BlockMix of the filling label (lo_f, hi_f) and
// BlockMix(X ^ V[j]) of the mixing label (lo_m, hi_m), interleaved.
template <int ROT, int DR_UNROLL>
PD_HD void blockmix_r1_dual(uint32_t (&lo_f)[16], uint32_t (&hi_f)[16], uint32_t (&lo_m)[16], uint32_t (&hi_m)[16],
                            const uint32_t (&vlo)[16], const uint32_t (&vhi)[16]) {
#pragma unroll
    for (int i = 0; i < 16; i++) {
        lo_f[i] ^= hi_f[i];
        hi_m[i] ^= vhi[i]; lo_m[i] = lo_m[i] ^ vlo[i] ^ hi_m[i];
    }
    chacha20_8_x2<ROT, DR_UNROLL>(lo_f, lo_m);
#pragma unroll
    for (int i = 0; i < 16; i++) { hi_f[i] ^= lo_f[i]; hi_m[i] ^= lo_m[i]; }
    chacha20_8_x2<ROT, DR_UNROLL>(hi_f, hi_m);
}

// BlockMix of two independent labels (a, b) in one instruction stream: the fill step of the phased ROMix kernel,
// where every thread writes the scratchpads of two labels of the same layer together.
template <int ROT, int DR_UNROLL>
PD_HD void blockmix_r1_x2(uint32_t (&lo_a)[16], uint32_t (&hi_a)[16], uint32_t (&lo_b)[16], uint32_t (&hi_b)[16]) {
#pragma unroll
    for (int i = 0; i < 16; i++) { lo_a[i] ^= hi_a[i]; lo_b[i] ^= hi_b[i]; }
    chacha20_8_x2<ROT, DR_UNROLL>(lo_a, lo_b);
#pragma unroll
    for (int i = 0; i < 16; i++) { hi_a[i] ^= lo_a[i]; hi_b[i] ^= lo_b[i]; }
    chacha20_8_x2<ROT, DR_UNROLL>(hi_a, hi_b);
}

// ------------------------------------------------------------------------------------------------
// Keccak-f[1600] (the Keccak submission §1.2; lane (x, y) at s[x + 5y]) and the label's two PBKDF2 passes.
// 13 permutations per label against 32768 ChaCha cores: ~0.5 % of the work, so the round loop stays rolled.
// ------------------------------------------------------------------------------------------------
#define PD_KECCAK_RC_TABLE \
    0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808aull, 0x8000000080008000ull, 0x000000000000808bull, \
    0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull, 0x000000000000008aull, 0x0000000000000088ull, \
    0x0000000080008009ull, 0x000000008000000aull, 0x000000008000808bull, 0x800000000000008bull, 0x8000000000008089ull, \
    0x8000000000008003ull, 0x8000000000008002ull, 0x8000000000000080ull, 0x000000000000800aull, 0x800000008000000aull, \
    0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull, 0x8000000080008008ull
static const uint64_t h_KeccakRC[24] = {PD_KECCAK_RC_TABLE};
#if defined(__CUDACC__)
static __device__ __constant__ uint64_t c_KeccakRC[24] = {PD_KECCAK_RC_TABLE};
#endif
PD_HD uint64_t keccak_rc(int i) {
#if defined(__CUDA_ARCH__)
    return c_KeccakRC[i];
#else
    return h_KeccakRC[i];
#endif
}
PD_HD uint64_t rotl64(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }   // 0 < k < 64

PD_HD void keccak_f1600(uint64_t (&s)[25]) {
#pragma unroll 1
    for (int round = 0; round < 24; round++) {
        // theta
        const uint64_t c0 = s[0] ^ s[5] ^ s[10] ^ s[15] ^ s[20], c1 = s[1] ^ s[6] ^ s[11] ^ s[16] ^ s[21],
                       c2 = s[2] ^ s[7] ^ s[12] ^ s[17] ^ s[22], c3 = s[3] ^ s[8] ^ s[13] ^ s[18] ^ s[23],
                       c4 = s[4] ^ s[9] ^ s[14] ^ s[19] ^ s[24];
        const uint64_t d0 = c4 ^ rotl64(c1, 1), d1 = c0 ^ rotl64(c2, 1), d2 = c1 ^ rotl64(c3, 1),
                       d3 = c2 ^ rotl64(c4, 1), d4 = c3 ^ rotl64(c0, 1);
#pragma unroll
        for (int y = 0; y < 25; y += 5) { s[y] ^= d0; s[y + 1] ^= d1; s[y + 2] ^= d2; s[y + 3] ^= d3; s[y + 4] ^= d4; }
        // rho + pi along the single 24-cycle of pi, starting from lane (1, 0)
        uint64_t t = s[1], u;
#define PD_RP(j, r) u = s[j]; s[j] = rotl64(t, r); t = u;
        PD_RP(10, 1) PD_RP(7, 3) PD_RP(11, 6) PD_RP(17, 10) PD_RP(18, 15) PD_RP(3, 21) PD_RP(5, 28) PD_RP(16, 36)
        PD_RP(8, 45) PD_RP(21, 55) PD_RP(24, 2) PD_RP(4, 14) PD_RP(15, 27) PD_RP(23, 41) PD_RP(19, 56) PD_RP(13, 8)
        PD_RP(12, 25) PD_RP(2, 43) PD_RP(20, 62) PD_RP(14, 18) PD_RP(22, 39) PD_RP(9, 61) PD_RP(6, 20) PD_RP(1, 44)
#undef PD_RP
        // chi
#pragma unroll
        for (int y = 0; y < 25; y += 5) {
            const uint64_t b0 = s[y], b1 = s[y + 1], b2 = s[y + 2], b3 = s[y + 3], b4 = s[y + 4];
            s[y] = b0 ^ (~b1 & b2); s[y + 1] = b1 ^ (~b2 & b3); s[y + 2] = b2 ^ (~b3 & b4);
            s[y + 3] = b3 ^ (~b4 & b0); s[y + 4] = b4 ^ (~b0 & b1);
        }
        s[0] ^= keccak_rc(round);   // iota
    }
}

// The HMAC key of label `index` is the scrypt password commitment || LE64(index) || 0^32: 72 bytes, exactly one
// Keccak-512 block (rate = 72), so it is used unhashed and K ^ pad fills the first sponge block.
// `c` = the commitment as 8 little-endian words.
constexpr uint64_t PD_IPAD = 0x3636363636363636ull, PD_OPAD = 0x5c5c5c5c5c5c5c5cull;
PD_HD void hmac_key_block(uint64_t (&s)[25], const uint32_t (&c)[8], uint64_t index, uint64_t pad) {
#pragma unroll
    for (int i = 0; i < 4; i++) s[i] = ((uint64_t)c[2 * i] | ((uint64_t)c[2 * i + 1] << 32)) ^ pad;
    s[4] = index ^ pad;
#pragma unroll
    for (int i = 5; i < 9; i++) s[i] = pad;
#pragma unroll
    for (int i = 9; i < 25; i++) s[i] = 0;
    keccak_f1600(s);
}
// outer hash of HMAC: H((K ^ opad) || digest), digest = 64 bytes = lanes 0..7, then pad 0x01 ... 0x80 in lane 8
PD_HD void hmac_outer(uint64_t (&s)[25], const uint32_t (&c)[8], uint64_t index, const uint64_t (&digest)[8]) {
    hmac_key_block(s, c, index, PD_OPAD);
#pragma unroll
    for (int i = 0; i < 8; i++) s[i] ^= digest[i];
    s[8] ^= 0x8000000000000001ull;
    keccak_f1600(s);
}

// PBKDF2-HMAC-Keccak512(P = key, S = "", c = 1, dkLen = 128) -> X as 32 LE words (scrypt step 1):
// T_k = HMAC(key, INT32BE(k)), k = 1, 2; T_1 -> lo, T_2 -> hi.  8 permutations.
PD_HD void label_expand(const uint32_t (&c)[8], uint64_t index, uint32_t (&lo)[16], uint32_t (&hi)[16]) {
#pragma unroll 1
    for (int k = 1; k <= 2; k++) {
        uint64_t s[25], d[8];
        hmac_key_block(s, c, index, PD_IPAD);
        s[0] ^= ((uint64_t)k << 24) | (1ull << 32);     // bytes 00 00 00 k, then the 0x01 pad byte
        s[8] ^= 0x8000000000000000ull;                  // final bit of the padding, byte 71
        keccak_f1600(s);
#pragma unroll
        for (int i = 0; i < 8; i++) d[i] = s[i];
        hmac_outer(s, c, index, d);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            // static indexing only: k is a runtime loop variable, so select with predicates
            if (k == 1) { lo[2 * i] = (uint32_t)s[i]; lo[2 * i + 1] = (uint32_t)(s[i] >> 32); }
            else { hi[2 * i] = (uint32_t)s[i]; hi[2 * i + 1] = (uint32_t)(s[i] >> 32); }
        }
    }
}

// PBKDF2-HMAC-Keccak512(P = key, S = X (128 bytes), c = 1, dkLen = 32) (scrypt step 3) -> the 32 output bytes as
// 8 BIG-endian words (out_be[0] holds bytes 0..3), the form the VRF comparison wants.  5 permutations.
PD_HD void label_final(const uint32_t (&c)[8], uint64_t index, const uint32_t (&lo)[16], const uint32_t (&hi)[16],
                       uint32_t (&out_be)[8]) {
    uint64_t s[25], d[8];
    hmac_key_block(s, c, index, PD_IPAD);
    // inner message after the key block: X (lanes x0..x15) || 00 00 00 01 -> block A = x0..x8, block B = x9..x15, counter
#pragma unroll
    for (int i = 0; i < 8; i++) s[i] ^= (uint64_t)lo[2 * i] | ((uint64_t)lo[2 * i + 1] << 32);
    s[8] ^= (uint64_t)hi[0] | ((uint64_t)hi[1] << 32);
    keccak_f1600(s);
#pragma unroll
    for (int i = 0; i < 7; i++) s[i] ^= (uint64_t)hi[2 * i + 2] | ((uint64_t)hi[2 * i + 3] << 32);
    s[7] ^= (1ull << 24) | (1ull << 32);
    s[8] ^= 0x8000000000000000ull;
    keccak_f1600(s);
#pragma unroll
    for (int i = 0; i < 8; i++) d[i] = s[i];
    hmac_outer(s, c, index, d);
#pragma unroll
    for (int i = 0; i < 4; i++) { out_be[2 * i] = bswap32((uint32_t)s[i]); out_be[2 * i + 1] = bswap32((uint32_t)(s[i] >> 32)); }
}

// ------------------------------------------------------------------------------------------------
// SHA-256 (FIPS 180-4 §6.2).  One compression of a 16-word big-endian block `w` into `st`.
// The round loop is 4 x 16 with a register ring so that code size stays small.  Used by the PoET proof-of-work
// search (poet_pow.cu); the label path does not use SHA-256.
// ------------------------------------------------------------------------------------------------
#define PD_K256_TABLE \
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, \
    0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, \
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, \
    0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, \
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, \
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, \
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, \
    0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2
static const uint32_t h_K256[64] = {PD_K256_TABLE};
#if defined(__CUDACC__)
static __device__ __constant__ uint32_t c_K256[64] = {PD_K256_TABLE};
#endif

PD_HD uint32_t sha_k(int i) {
#if defined(__CUDA_ARCH__)
    return c_K256[i];
#else
    return h_K256[i];
#endif
}
PD_HD uint32_t rotr(uint32_t x, int k) { return rotl(x, 32 - k); }

PD_HD void sha256_compress(uint32_t (&st)[8], uint32_t (&w)[16]) {
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll 1
    for (int base = 0; base < 64; base += 16) {
#pragma unroll
        for (int t = 0; t < 16; t++) {
            if (base) {
                const uint32_t w15 = w[(t + 1) & 15], w2 = w[(t + 14) & 15];
                const uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ (w15 >> 3);
                const uint32_t s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ (w2 >> 10);
                w[t] = w[t] + s0 + w[(t + 9) & 15] + s1;
            }
            const uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
            const uint32_t ch = (e & f) ^ (~e & g);
            const uint32_t t1 = h + S1 + ch + sha_k(base + t) + w[t];
            const uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
            const uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
            h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + S0 + mj;
        }
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

PD_HD void sha256_iv(uint32_t (&st)[8]) {
    st[0] = 0x6a09e667; st[1] = 0xbb67ae85; st[2] = 0x3c6ef372; st[3] = 0xa54ff53a;
    st[4] = 0x510e527f; st[5] = 0x9b05688c; st[6] = 0x1f83d9ab; st[7] = 0x5be0cd19;
}

// ------------------------------------------------------------------------------------------------
// VRF order: lexicographic (label_be[0..7], index) "a < b", label32 as eight big-endian words.  With equal indices
// (0, 0) it is the strict "label32 < threshold" of the VRF-nonce rule (K3's candidates, K4, K9).
// ------------------------------------------------------------------------------------------------
PD_HD bool cand_less(const uint32_t (&a)[8], uint64_t ai, const uint32_t (&b)[8], uint64_t bi) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
        if (a[k] != b[k]) return a[k] < b[k];
    }
    return ai < bi;
}

}  // namespace b200post
