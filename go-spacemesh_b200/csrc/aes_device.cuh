// aes_device.cuh — AES-128 single-block encryption for sm_90a kernels (FIPS-197, T-table form).
//
// Used by the verify epilogue and the proving scan: one 16-byte label is encrypted under a per-proof key and
// ciphertext bytes are compared with the proving difficulty (ASSUMED post-rs Prover8_56 scheme, see
// include/b200post_verify.h).  Round keys are expanded on the host (AES-NI) and read as 11 x uint4.
//
// State words are little-endian columns (byte 0 = row 0).  One table T0 (T0[x] = {2·S[x], S[x], S[x], 3·S[x]})
// lives in shared memory, REPLICATED PER LANE (entry x of lane l at word x*32 + l): every lane owns bank l, so
// the 160 data-dependent lookups of an encryption are bank-conflict-free by construction (a single shared
// copy would serialise ~3.5 lanes per bank on random bytes).  T1..T3 are byte rotations of T0 (one PRMT each)
// and the last round takes S[x] from byte 1 of T0[x].  32 KiB of shared memory per CTA.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace b200post {

struct AesTables { uint32_t t0[256]; uint8_t sbox[256]; };   // host-built once, uploaded to global memory

// fills `t` (host): S-box from the GF(2^8) inverse + affine map, then the MixColumns-folded table
inline void aes_build_tables(AesTables &t) {
    auto xtime = [](uint8_t a) { return (uint8_t)((a << 1) ^ ((a & 0x80) ? 0x1b : 0)); };
    // log/antilog over generator 3
    uint8_t exp[256], log[256];
    uint8_t x = 1;
    for (int i = 0; i < 255; i++) { exp[i] = x; log[x] = (uint8_t)i; x = (uint8_t)(x ^ xtime(x)); }
    exp[255] = exp[0];
    for (int v = 0; v < 256; v++) {
        const uint8_t inv = v ? exp[(255 - log[v]) % 255] : 0;
        uint8_t s = inv, r = inv;
        for (int k = 0; k < 4; k++) { r = (uint8_t)((r << 1) | (r >> 7)); s ^= r; }
        s ^= 0x63;
        t.sbox[v] = s;
        const uint8_t s2 = xtime(s), s3 = (uint8_t)(s2 ^ s);
        t.t0[v] = (uint32_t)s2 | ((uint32_t)s << 8) | ((uint32_t)s << 16) | ((uint32_t)s3 << 24);
    }
}

#if defined(__CUDACC__)
constexpr int AES_SMEM_BYTES = 256 * 32 * 4;   // dynamic shared memory a kernel using these functions needs

// copy T0 into the lane-replicated shared image; every thread of the CTA must call it
__device__ __forceinline__ void aes_load_smem(uint32_t *sm, const AesTables *__restrict__ g) {
    for (int i = threadIdx.x; i < 256 * 32; i += blockDim.x) sm[i] = g->t0[i >> 5];
    __syncthreads();
}

__device__ __forceinline__ uint32_t rotl8(uint32_t v) { return __byte_perm(v, 0, 0x2103); }    // T1 from T0
__device__ __forceinline__ uint32_t rotl16(uint32_t v) { return __byte_perm(v, 0, 0x1032); }   // T2
__device__ __forceinline__ uint32_t rotl24(uint32_t v) { return __byte_perm(v, 0, 0x0321); }   // T3

// out = AES-128-Encrypt(rk, in); rk = 11 round keys as little-endian column words; tl = sm + lane
__device__ __forceinline__ uint4 aes128_encrypt(const uint32_t *__restrict__ tl, const uint4 *__restrict__ rk, uint4 in) {
#define AES_T(x) tl[(x) << 5]
    uint4 k = rk[0];
    uint32_t s0 = in.x ^ k.x, s1 = in.y ^ k.y, s2 = in.z ^ k.z, s3 = in.w ^ k.w;
#pragma unroll
    for (int r = 1; r < 10; r++) {
        k = rk[r];
        const uint32_t t0 = AES_T(s0 & 0xff) ^ rotl8(AES_T((s1 >> 8) & 0xff)) ^ rotl16(AES_T((s2 >> 16) & 0xff)) ^ rotl24(AES_T(s3 >> 24)) ^ k.x;
        const uint32_t t1 = AES_T(s1 & 0xff) ^ rotl8(AES_T((s2 >> 8) & 0xff)) ^ rotl16(AES_T((s3 >> 16) & 0xff)) ^ rotl24(AES_T(s0 >> 24)) ^ k.y;
        const uint32_t t2 = AES_T(s2 & 0xff) ^ rotl8(AES_T((s3 >> 8) & 0xff)) ^ rotl16(AES_T((s0 >> 16) & 0xff)) ^ rotl24(AES_T(s1 >> 24)) ^ k.z;
        const uint32_t t3 = AES_T(s3 & 0xff) ^ rotl8(AES_T((s0 >> 8) & 0xff)) ^ rotl16(AES_T((s1 >> 16) & 0xff)) ^ rotl24(AES_T(s2 >> 24)) ^ k.w;
        s0 = t0; s1 = t1; s2 = t2; s3 = t3;
    }
    k = rk[10];
    // last round: SubBytes + ShiftRows only; S[x] is byte 1 of T0[x].  PRMT picks byte 1 of four lookups.
#define AES_S4(a, b, c, d) \
    (__byte_perm(__byte_perm(AES_T((a) & 0xff), AES_T(((b) >> 8) & 0xff), 0x0051), __byte_perm(AES_T(((c) >> 16) & 0xff), AES_T((d) >> 24), 0x0051), 0x5410))
    uint4 o;
    o.x = AES_S4(s0, s1, s2, s3) ^ k.x;
    o.y = AES_S4(s1, s2, s3, s0) ^ k.y;
    o.z = AES_S4(s2, s3, s0, s1) ^ k.z;
    o.w = AES_S4(s3, s0, s1, s2) ^ k.w;
#undef AES_S4
#undef AES_T
    return o;
}
__device__ __forceinline__ uint32_t uint4_byte(const uint4 &v, uint32_t i) {
    const uint32_t w = i < 4 ? v.x : i < 8 ? v.y : i < 12 ? v.z : v.w;
    return (w >> (8 * (i & 3))) & 0xff;
}
#endif

}  // namespace b200post
