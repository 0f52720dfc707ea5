// randomx_kernels.cu — RandomX (k2pow) on sm_90a.  go-spacemesh reaches this function only through an RPC to the
// external post-service (activation/nipost.go:171) and through libpost's verifier (activation/post_verifier.go:159);
// the arithmetic is tevador/RandomX v1.1.x (doc/specs.md), restated here for the GPU:
//
//   dataset      one thread per 64-byte item: 8 SuperscalarHash programs (identical for every item, so a warp never
//                diverges) over registers held in shared memory, 8 random 64-byte reads of the 256 MiB cache (spec §7.3)
//   seed         Blake2b-512 of the 48-byte k2pow input (or of caller-supplied inputs), one thread per VM
//   fill         AesGenerator1R: four lanes per VM (one per AES column), 32768 chained rounds each, T-tables in smem
//   program      AesGenerator4R -> configuration + 256 instructions, decoded to an 8-byte form (spec §4.5, §5)
//   execute      the VM.  One thread per VM, its 256-byte register file in shared memory ([slot][thread], conflict
//                free), its decoded program in HBM as [pc][vm] (a warp in step reads 256 contiguous bytes), its 2 MiB
//                scratchpad private in HBM.  Operand fetch, the one scratchpad load and the write-back are common code;
//                only the ALU step of each instruction sits in the divergent switch.  FP rounding modes are per VM:
//                add/mul use the hardware's static-rounding instructions, div/sqrt round to nearest and are corrected
//                by the sign of the exact FMA residual (no 4-way divergence over ~100-instruction software routines).
//   chain seed   Blake2b-512 of the register file;  finalize: AesHash1R over the scratchpad + Blake2b-256.
//
// Throughput is bounded by dependent scratchpad accesses (one 8-byte access per ~5 instructions, each a random HBM
// sector) and by SIMT divergence across VMs — RandomX is built to be that — so the lever the GPU offers is capacity:
// thousands of 2 MiB scratchpads resident in 80 GB of HBM and the full 2080 MiB dataset next to them.
#include "randomx_kernels.cuh"

#include <cstring>

namespace b200post {
namespace rx {
namespace {

using u64 = uint64_t;
using u32 = uint32_t;

// ---------------------------------------------------------------------------------------------- tables
__device__ u32 g_te0[256], g_td0[256];      // AES round tables (enc: {2s, s, s, 3s}; dec: {14i, 9i, 13i, 11i}), byte 0 = row 0
__device__ uint8_t g_opmap[256];            // opcode byte -> instruction type (spec table 5.1 frequencies)
__constant__ uint8_t c_sigma[12][16] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
    {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
    {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
    {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
    {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};
__constant__ u64 c_b2iv[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                              0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
// generator keys / hash state: Blake2b of fixed strings (spec §3.2-3.4), derived on the host at upload time
__constant__ u32 c_gen1_keys[16], c_gen4_keys[32], c_hash_state[16], c_hash_xkeys[8];

// ---------------------------------------------------------------------------------------------- Blake2b
__device__ __forceinline__ u64 ror64(u64 v, int n) { return (v >> n) | (v << (64 - n)); }

__device__ void b2_compress(u64 h[8], const u64 m[16], u64 t, bool last) {
    u64 v[16];
#pragma unroll
    for (int i = 0; i < 8; i++) { v[i] = h[i]; v[i + 8] = c_b2iv[i]; }
    v[12] ^= t;
    if (last) v[14] = ~v[14];
#define B2G(r, i, a, b, c, d)                                             \
    a = a + b + m[c_sigma[r][2 * i]];     d = ror64(d ^ a, 32);           \
    c = c + d;                            b = ror64(b ^ c, 24);           \
    a = a + b + m[c_sigma[r][2 * i + 1]]; d = ror64(d ^ a, 16);           \
    c = c + d;                            b = ror64(b ^ c, 63);
    for (int r = 0; r < 12; r++) {
        B2G(r, 0, v[0], v[4], v[8], v[12]) B2G(r, 1, v[1], v[5], v[9], v[13])
        B2G(r, 2, v[2], v[6], v[10], v[14]) B2G(r, 3, v[3], v[7], v[11], v[15])
        B2G(r, 4, v[0], v[5], v[10], v[15]) B2G(r, 5, v[1], v[6], v[11], v[12])
        B2G(r, 6, v[2], v[7], v[8], v[13]) B2G(r, 7, v[3], v[4], v[9], v[14])
    }
#undef B2G
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[i + 8];
}
__device__ __forceinline__ void b2_init(u64 h[8], u32 outlen) {
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = c_b2iv[i];
    h[0] ^= 0x01010000ull ^ outlen;
}

// ---------------------------------------------------------------------------------------------- AES rounds
struct AesSmem { u32 te[256], td[256]; };
__device__ __forceinline__ void aes_load(AesSmem &sm) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) { sm.te[i] = g_te0[i]; sm.td[i] = g_td0[i]; }
    __syncthreads();
}
__device__ __forceinline__ u32 rl8(u32 v) { return __byte_perm(v, 0, 0x2103); }
__device__ __forceinline__ u32 rl16(u32 v) { return __byte_perm(v, 0, 0x1032); }
__device__ __forceinline__ u32 rl24(u32 v) { return __byte_perm(v, 0, 0x0321); }
// x86 AESENC: ShiftRows, SubBytes, MixColumns, xor key.  s = 4 little-endian column words.
__device__ __forceinline__ void aes_enc(const AesSmem &sm, u32 s[4], const u32 k[4]) {
    const u32 t0 = sm.te[s[0] & 255] ^ rl8(sm.te[(s[1] >> 8) & 255]) ^ rl16(sm.te[(s[2] >> 16) & 255]) ^ rl24(sm.te[s[3] >> 24]);
    const u32 t1 = sm.te[s[1] & 255] ^ rl8(sm.te[(s[2] >> 8) & 255]) ^ rl16(sm.te[(s[3] >> 16) & 255]) ^ rl24(sm.te[s[0] >> 24]);
    const u32 t2 = sm.te[s[2] & 255] ^ rl8(sm.te[(s[3] >> 8) & 255]) ^ rl16(sm.te[(s[0] >> 16) & 255]) ^ rl24(sm.te[s[1] >> 24]);
    const u32 t3 = sm.te[s[3] & 255] ^ rl8(sm.te[(s[0] >> 8) & 255]) ^ rl16(sm.te[(s[1] >> 16) & 255]) ^ rl24(sm.te[s[2] >> 24]);
    s[0] = t0 ^ k[0]; s[1] = t1 ^ k[1]; s[2] = t2 ^ k[2]; s[3] = t3 ^ k[3];
}
// x86 AESDEC: InvShiftRows, InvSubBytes, InvMixColumns, xor key
__device__ __forceinline__ void aes_dec(const AesSmem &sm, u32 s[4], const u32 k[4]) {
    const u32 t0 = sm.td[s[0] & 255] ^ rl8(sm.td[(s[3] >> 8) & 255]) ^ rl16(sm.td[(s[2] >> 16) & 255]) ^ rl24(sm.td[s[1] >> 24]);
    const u32 t1 = sm.td[s[1] & 255] ^ rl8(sm.td[(s[0] >> 8) & 255]) ^ rl16(sm.td[(s[3] >> 16) & 255]) ^ rl24(sm.td[s[2] >> 24]);
    const u32 t2 = sm.td[s[2] & 255] ^ rl8(sm.td[(s[1] >> 8) & 255]) ^ rl16(sm.td[(s[0] >> 16) & 255]) ^ rl24(sm.td[s[3] >> 24]);
    const u32 t3 = sm.td[s[3] & 255] ^ rl8(sm.td[(s[2] >> 8) & 255]) ^ rl16(sm.td[(s[1] >> 16) & 255]) ^ rl24(sm.td[s[0] >> 24]);
    s[0] = t0 ^ k[0]; s[1] = t1 ^ k[1]; s[2] = t2 ^ k[2]; s[3] = t3 ^ k[3];
}

// ---------------------------------------------------------------------------------------------- dataset
__device__ __forceinline__ u64 mulh_u(u64 a, u64 b) { return __umul64hi(a, b); }
__device__ __forceinline__ u64 mulh_s(u64 a, u64 b) { return (u64)__mul64hi((long long)a, (long long)b); }
__device__ __forceinline__ u64 sext(u32 v) { return (u64)(long long)(int)v; }

constexpr int kDatasetThreads = 256;
struct SsArgs { const SsOp *ops; u32 first[kCacheAccesses + 1]; u32 address_reg[kCacheAccesses]; };

__global__ void __launch_bounds__(kDatasetThreads) dataset_kernel(const u64 *__restrict__ cache, SsArgs ss, u64 *__restrict__ dataset,
                                                                   u64 first_item, u64 count) {
    __shared__ u64 regs[8][kDatasetThreads];
    const u64 idx = (u64)blockIdx.x * kDatasetThreads + threadIdx.x;
    if (idx >= count) return;
    const u64 item = first_item + idx;
    const int t = threadIdx.x;
    const u64 r0 = (item + 1) * 6364136223846793005ull;
    regs[0][t] = r0;
    regs[1][t] = r0 ^ 9298411001130361340ull;  regs[2][t] = r0 ^ 12065312585734608966ull;
    regs[3][t] = r0 ^ 9306329213124626780ull;  regs[4][t] = r0 ^ 5281919268842080866ull;
    regs[5][t] = r0 ^ 10536153434571861004ull; regs[6][t] = r0 ^ 3398623926847679864ull;
    regs[7][t] = r0 ^ 9549104520008361294ull;
    u64 line = item;
    constexpr u64 kLineMask = (u64)kCacheKiB * 1024 / 64 - 1;
    for (int p = 0; p < (int)kCacheAccesses; p++) {
        const ulonglong2 *mix = reinterpret_cast<const ulonglong2 *>(cache + (line & kLineMask) * 8);
        ulonglong2 m0 = __ldg(mix), m1 = __ldg(mix + 1), m2 = __ldg(mix + 2), m3 = __ldg(mix + 3);   // in flight under the program
        for (u32 j = ss.first[p]; j < ss.first[p + 1]; j++) {
            const uint4 raw = __ldg(reinterpret_cast<const uint4 *>(ss.ops + j));   // warp-uniform address: one broadcast
            const u32 op = raw.x & 255, dst = (raw.x >> 8) & 255, src = (raw.x >> 16) & 255, shift = raw.x >> 24;
            const u64 d = regs[dst][t], s = regs[src][t];
            u64 res;
            switch (op) {
                case SS_ISUB_R: res = d - s; break;
                case SS_IXOR_R: res = d ^ s; break;
                case SS_IADD_RS: res = d + (s << shift); break;
                case SS_IMUL_R: res = d * s; break;
                case SS_IROR_C: res = ror64(d, raw.y & 63); break;   // imm is 1..63
                case SS_IADD_C: res = d + sext(raw.y); break;
                case SS_IXOR_C: res = d ^ sext(raw.y); break;
                case SS_IMULH_R: res = mulh_u(d, s); break;
                case SS_ISMULH_R: res = mulh_s(d, s); break;
                default: res = d * (((u64)raw.w << 32) | raw.z); break;   // SS_IMUL_RCP
            }
            regs[dst][t] = res;
        }
        regs[0][t] ^= m0.x; regs[1][t] ^= m0.y; regs[2][t] ^= m1.x; regs[3][t] ^= m1.y;
        regs[4][t] ^= m2.x; regs[5][t] ^= m2.y; regs[6][t] ^= m3.x; regs[7][t] ^= m3.y;
        line = regs[ss.address_reg[p]][t];
    }
    ulonglong2 *out = reinterpret_cast<ulonglong2 *>(dataset + item * 8);
    out[0] = make_ulonglong2(regs[0][t], regs[1][t]); out[1] = make_ulonglong2(regs[2][t], regs[3][t]);
    out[2] = make_ulonglong2(regs[4][t], regs[5][t]); out[3] = make_ulonglong2(regs[6][t], regs[7][t]);
}

// ---------------------------------------------------------------------------------------------- seeds
__global__ void seed_inputs_kernel(u64 *__restrict__ seed, u32 stride, u32 n, const uint8_t *__restrict__ inputs, u32 len) {
    const u32 vm = blockIdx.x * blockDim.x + threadIdx.x;
    if (vm >= n) return;
    const uint8_t *in = inputs + (size_t)vm * len;
    u64 h[8], m[16];
    b2_init(h, 64);
    u32 off = 0;
    while (len - off > 128) {
        for (int i = 0; i < 16; i++) { u64 w = 0; for (int b = 0; b < 8; b++) w |= (u64)in[off + 8 * i + b] << (8 * b); m[i] = w; }
        off += 128;
        b2_compress(h, m, off, false);
    }
    for (int i = 0; i < 16; i++) { u64 w = 0; for (int b = 0; b < 8; b++) { const u32 p = off + 8 * i + b; if (p < len) w |= (u64)in[p] << (8 * b); } m[i] = w; }
    b2_compress(h, m, len, true);
    for (int i = 0; i < 8; i++) seed[(size_t)i * stride + vm] = h[i];
}
__global__ void seed_k2pow_kernel(u64 *__restrict__ seed, u32 stride, u32 n, K2powTemplate t) {
    const u32 vm = blockIdx.x * blockDim.x + threadIdx.x;
    if (vm >= n) return;
    uint8_t in[48];
    const u64 pow = t.start + vm;
    for (int i = 0; i < 7; i++) in[i] = (uint8_t)(pow >> (8 * i));
    for (int i = 0; i < 41; i++) in[7 + i] = t.tail[i];
    u64 h[8], m[16];
    b2_init(h, 64);
    for (int i = 0; i < 16; i++) { u64 w = 0; if (i < 6) for (int b = 0; b < 8; b++) w |= (u64)in[8 * i + b] << (8 * b); m[i] = w; }
    b2_compress(h, m, 48, true);
    for (int i = 0; i < 8; i++) seed[(size_t)i * stride + vm] = h[i];
}

// ---------------------------------------------------------------------------------------------- scratchpad fill / hash
// 4 lanes per VM: lane c owns AES column c of the 64-byte generator state (columns 0,2 decrypt, 1,3 encrypt)
__global__ void __launch_bounds__(256) fill_kernel(u64 *__restrict__ seed, u32 stride, u32 n, uint8_t *__restrict__ scratchpads, uint8_t *__restrict__ hot) {
    __shared__ AesSmem sm;
    aes_load(sm);
    const u32 gid = blockIdx.x * blockDim.x + threadIdx.x, vm = gid >> 2, col = gid & 3;
    if (vm >= n) return;
    u32 s[4], k[4];
    { const u64 a = seed[(size_t)(2 * col) * stride + vm], b = seed[(size_t)(2 * col + 1) * stride + vm];
      s[0] = (u32)a; s[1] = (u32)(a >> 32); s[2] = (u32)b; s[3] = (u32)(b >> 32); }
#pragma unroll
    for (int i = 0; i < 4; i++) k[i] = c_gen1_keys[4 * col + i];
    uint4 *out = reinterpret_cast<uint4 *>(scratchpads + (size_t)vm * kScratchpadL3) + col;
    uint4 *out_hot = reinterpret_cast<uint4 *>(hot + (size_t)vm * kScratchpadL1) + col;   // the first 16 KiB live in the hot plane
    const bool dec = (col & 1) == 0;
    for (u32 i = 0; i < kScratchpadL3 / 64; i++) {
        if (dec) aes_dec(sm, s, k); else aes_enc(sm, s, k);
        (i < kScratchpadL1 / 64 ? out_hot : out)[4 * (size_t)i] = make_uint4(s[0], s[1], s[2], s[3]);
    }
    seed[(size_t)(2 * col) * stride + vm] = (u64)s[0] | ((u64)s[1] << 32);
    seed[(size_t)(2 * col + 1) * stride + vm] = (u64)s[2] | ((u64)s[3] << 32);
}
// AesHash1R: the scratchpad is the key stream (columns 0,2 encrypt, 1,3 decrypt), two fixed finishing rounds -> a0..a3
__global__ void __launch_bounds__(256) hash_scratchpad_kernel(u64 *__restrict__ regfile, u32 stride, u32 n, const uint8_t *__restrict__ scratchpads, const uint8_t *__restrict__ hot) {
    __shared__ AesSmem sm;
    aes_load(sm);
    const u32 gid = blockIdx.x * blockDim.x + threadIdx.x, vm = gid >> 2, col = gid & 3;
    if (vm >= n) return;
    u32 s[4];
#pragma unroll
    for (int i = 0; i < 4; i++) s[i] = c_hash_state[4 * col + i];
    const uint4 *in_cold = reinterpret_cast<const uint4 *>(scratchpads + (size_t)vm * kScratchpadL3) + col;
    const uint4 *in_hot = reinterpret_cast<const uint4 *>(hot + (size_t)vm * kScratchpadL1) + col;
    auto key_at = [&](u32 i) { return (i < kScratchpadL1 / 64 ? in_hot : in_cold)[4 * (size_t)i]; };
    const bool enc = (col & 1) == 0;
    constexpr u32 kRounds = kScratchpadL3 / 64;
    uint4 nxt[4];
#pragma unroll
    for (int j = 0; j < 4; j++) nxt[j] = key_at(j);
    for (u32 i = 0; i < kRounds; i += 4) {
        uint4 cur[4];
#pragma unroll
        for (int j = 0; j < 4; j++) { cur[j] = nxt[j]; if (i + 4 + j < kRounds) nxt[j] = key_at(i + 4 + j); }   // keys do not depend on the state: prefetch
#pragma unroll
        for (int j = 0; j < 4; j++) { const u32 k[4] = {cur[j].x, cur[j].y, cur[j].z, cur[j].w}; if (enc) aes_enc(sm, s, k); else aes_dec(sm, s, k); }
    }
#pragma unroll
    for (int r = 0; r < 2; r++) { const u32 k[4] = {c_hash_xkeys[4 * r], c_hash_xkeys[4 * r + 1], c_hash_xkeys[4 * r + 2], c_hash_xkeys[4 * r + 3]}; if (enc) aes_enc(sm, s, k); else aes_dec(sm, s, k); }
    regfile[(size_t)(24 + 2 * col) * stride + vm] = (u64)s[0] | ((u64)s[1] << 32);
    regfile[(size_t)(25 + 2 * col) * stride + vm] = (u64)s[2] | ((u64)s[3] << 32);
}

// ---------------------------------------------------------------------------------------------- program generation + decode
// instruction types in opcode order (spec table 5.1)
enum : uint8_t { T_IADD_RS, T_IADD_M, T_ISUB_R, T_ISUB_M, T_IMUL_R, T_IMUL_M, T_IMULH_R, T_IMULH_M, T_ISMULH_R, T_ISMULH_M, T_IMUL_RCP,
                 T_INEG_R, T_IXOR_R, T_IXOR_M, T_IROR_R, T_IROL_R, T_ISWAP_R, T_FSWAP_R, T_FADD_R, T_FADD_M, T_FSUB_R, T_FSUB_M,
                 T_FSCAL_R, T_FMUL_R, T_FDIV_M, T_FSQRT_R, T_CBRANCH, T_CFROUND, T_ISTORE, T_NOP, T_COUNT };
// Decoded instruction (8 bytes): word0 = (src slot * 8) | op << 8 | aux << 16 | (dst slot * 8) << 24, word1 = imm32.
// Dense opcodes, one per (operation, operand kind), so each handler touches only what it needs; slot fields are byte
// offsets into the register file in shared memory (slots: 0-7 r, 8-15 f lo/hi, 16-23 e lo/hi, 24-31 a lo/hi);
// aux = shift / rotate count / reciprocal slot / log2 of the scratchpad level size.
enum : uint8_t { W_NOP, W_IADD_RS, W_ISUB_R, W_IMUL_R, W_IMULH_R, W_ISMULH_R, W_IXOR_R, W_IROR_R, W_IROL_R, W_ISWAP,
                 W_ISUB_I, W_IMUL_I, W_IXOR_I, W_IROR_I, W_IROL_I, W_INEG, W_IMUL_RCP, W_IMUL_RCP_SLOW,
                 W_IADD_M, W_ISUB_M, W_IMUL_M, W_IMULH_M, W_ISMULH_M, W_IXOR_M,
                 W_IADD_A, W_ISUB_A, W_IMUL_A, W_IMULH_A, W_ISMULH_A, W_IXOR_A,
                 W_CBRANCH, W_CFROUND, W_ISTORE,
                 W_FSWAP, W_FADD_R, W_FSUB_R, W_FSCAL, W_FMUL_R, W_FSQRT, W_FADD_M, W_FSUB_M, W_FDIV_M,
                 W_END,       // sentinel the VM kernel appends after the 256th instruction: the program loop has no counter
                 W_COUNT };
__device__ __forceinline__ u32 wpack(u32 op, u32 dslot, u32 sslot, u32 aux) { return (sslot * 8) | (op << 8) | (aux << 16) | ((dslot * 8) << 24); }
constexpr u32 kL3Mask = (kScratchpadL3 - 1) & ~7u;
constexpr u32 kL3Mask64 = (kScratchpadL3 - 1) & ~63u;
constexpr u32 kDatasetAlignMask = (u32)((kDatasetBase - 1) & ~63ull);

__device__ u64 device_reciprocal(u32 divisor) {
    u64 q = (1ull << 63) / divisor, r = (1ull << 63) % divisor;
    const int bits = 32 - __clz(divisor);
    for (int i = 0; i < bits; i++) {
        if (r >= divisor - r) { q = 2 * q + 1; r = 2 * r - divisor; }
        else { q = 2 * q; r = 2 * r; }
    }
    return q;
}

__global__ void __launch_bounds__(128) program_kernel(BatchBuffers b, u32 n, bool first_program) {
    __shared__ AesSmem sm;
    __shared__ uint8_t opmap[256];
    __shared__ short usage[8][128];     // CBRANCH targets: last instruction that wrote each integer register
    aes_load(sm);
    for (int i = threadIdx.x; i < 256; i += blockDim.x) opmap[i] = g_opmap[i];
    __syncthreads();
    const u32 vm = blockIdx.x * blockDim.x + threadIdx.x, t = threadIdx.x;
    if (vm >= n) return;
    const u32 stride = b.stride;
    u32 st[4][4];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const u64 lo = b.seed[(size_t)(2 * c) * stride + vm], hi = b.seed[(size_t)(2 * c + 1) * stride + vm];
        st[c][0] = (u32)lo; st[c][1] = (u32)(lo >> 32); st[c][2] = (u32)hi; st[c][3] = (u32)(hi >> 32);
    }
    auto next64 = [&](u64 out[8]) {   // AesGenerator4R: columns 0,1 keys 0-3, columns 2,3 keys 4-7; 0,2 decrypt, 1,3 encrypt
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const u32 ka[4] = {c_gen4_keys[4 * k], c_gen4_keys[4 * k + 1], c_gen4_keys[4 * k + 2], c_gen4_keys[4 * k + 3]};
            const u32 kb[4] = {c_gen4_keys[16 + 4 * k], c_gen4_keys[17 + 4 * k], c_gen4_keys[18 + 4 * k], c_gen4_keys[19 + 4 * k]};
            aes_dec(sm, st[0], ka); aes_enc(sm, st[1], ka); aes_dec(sm, st[2], kb); aes_enc(sm, st[3], kb);
        }
#pragma unroll
        for (int c = 0; c < 4; c++) { out[2 * c] = (u64)st[c][0] | ((u64)st[c][1] << 32); out[2 * c + 1] = (u64)st[c][2] | ((u64)st[c][3] << 32); }
    };
    u64 ent[16];
    next64(ent); next64(ent + 8);
    // configuration (spec §4.5): a0-3 = small positive doubles, ma/mx, address registers, dataset offset, e masks
    constexpr u64 kMant = (1ull << 52) - 1;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const u64 e = ent[i];
        b.regfile[(size_t)(24 + i) * stride + vm] = ((((e >> 59) + 1023) & 2047) << 52) | (e & kMant);
    }
    const u32 ma = (u32)ent[8] & kDatasetAlignMask, mx = (u32)ent[10];
    b.config[(size_t)0 * stride + vm] = (u64)ma | ((u64)mx << 32);
    const u64 ds_off = (ent[13] % (kDatasetExtra / 64 + 1)) * 64;
    b.config[(size_t)1 * stride + vm] = ds_off | ((ent[12] & 15) << 60);
    auto fmask = [](u64 e) { return (e & ((1ull << 22) - 1)) | ((0x300ull | ((e >> 60) << 4)) << 52); };
    b.config[(size_t)2 * stride + vm] = fmask(ent[14]);
    b.config[(size_t)3 * stride + vm] = fmask(ent[15]);
    if (first_program) b.fprc[vm] = 0;

#pragma unroll
    for (int i = 0; i < 8; i++) usage[i][t] = -1;
    u32 n_rcp = 0;
    for (int chunk = 0; chunk < kProgramSize / 8; chunk++) {
        u64 raw[8];
        next64(raw);
        for (int j = 0; j < 8; j++) {
            const int i = chunk * 8 + j;
            const u32 lo = (u32)raw[j], imm = (u32)(raw[j] >> 32);
            const u32 type = opmap[lo & 255], dst = (lo >> 8) & 7, src = (lo >> 16) & 7, mod = lo >> 24;
            u32 w0 = W_NOP, w1 = imm;
            {
                const u32 bits12 = (mod & 3) ? 14 : 18;   // log2 of the level size: L1 16 KiB, L2 256 KiB (L3 2 MiB = 21)
                switch (type) {
                    case T_IADD_RS: w0 = wpack(W_IADD_RS, dst, src, (mod >> 2) & 3); w1 = dst == 5 ? imm : 0; usage[dst][t] = (short)i; break;
                    case T_IADD_M: case T_ISUB_M: case T_IMUL_M: case T_IMULH_M: case T_ISMULH_M: case T_IXOR_M: {
                        const u32 k = type == T_IADD_M ? 0 : type == T_ISUB_M ? 1 : type == T_IMUL_M ? 2 : type == T_IMULH_M ? 3 : type == T_ISMULH_M ? 4 : 5;
                        if (src != dst) w0 = wpack(W_IADD_M + k, dst, src, bits12);
                        else { w0 = wpack(W_IADD_A + k, dst, 0, 0); w1 = imm & kL3Mask; }       // constant address
                        usage[dst][t] = (short)i;
                    } break;
                    case T_ISUB_R: case T_IMUL_R: case T_IXOR_R: {
                        const u32 k = type == T_ISUB_R ? 0 : type == T_IMUL_R ? 1 : 2;
                        w0 = src != dst ? wpack((k == 0 ? W_ISUB_R : k == 1 ? W_IMUL_R : W_IXOR_R), dst, src, 0)
                                        : wpack((k == 0 ? W_ISUB_I : k == 1 ? W_IMUL_I : W_IXOR_I), dst, 0, 0);
                        usage[dst][t] = (short)i;
                    } break;
                    case T_IMULH_R: w0 = wpack(W_IMULH_R, dst, src, 0); usage[dst][t] = (short)i; break;
                    case T_ISMULH_R: w0 = wpack(W_ISMULH_R, dst, src, 0); usage[dst][t] = (short)i; break;
                    case T_IMUL_RCP:
                        if (imm & (imm - 1)) {
                            if (n_rcp < (u32)kRcpSlots) { b.rcp[(size_t)vm * kRcpSlots + n_rcp] = device_reciprocal(imm); w0 = wpack(W_IMUL_RCP, dst, 0, n_rcp); n_rcp++; }
                            else w0 = wpack(W_IMUL_RCP_SLOW, dst, 0, 0);
                            usage[dst][t] = (short)i;
                        }
                        break;
                    case T_INEG_R: w0 = wpack(W_INEG, dst, 0, 0); usage[dst][t] = (short)i; break;
                    case T_IROR_R: w0 = src != dst ? wpack(W_IROR_R, dst, src, 0) : wpack(W_IROR_I, dst, 0, imm & 63); usage[dst][t] = (short)i; break;
                    case T_IROL_R: w0 = src != dst ? wpack(W_IROL_R, dst, src, 0) : wpack(W_IROL_I, dst, 0, imm & 63); usage[dst][t] = (short)i; break;
                    case T_ISWAP_R: if (src != dst) { w0 = wpack(W_ISWAP, dst, src, 0); usage[dst][t] = (short)i; usage[src][t] = (short)i; } break;
                    case T_FSWAP_R: w0 = wpack(W_FSWAP, 8 + 2 * dst, 0, 0); break;
                    case T_FADD_R: w0 = wpack(W_FADD_R, 8 + 2 * (dst & 3), 24 + 2 * (src & 3), 0); break;
                    case T_FADD_M: w0 = wpack(W_FADD_M, 8 + 2 * (dst & 3), src, bits12); break;
                    case T_FSUB_R: w0 = wpack(W_FSUB_R, 8 + 2 * (dst & 3), 24 + 2 * (src & 3), 0); break;
                    case T_FSUB_M: w0 = wpack(W_FSUB_M, 8 + 2 * (dst & 3), src, bits12); break;
                    case T_FSCAL_R: w0 = wpack(W_FSCAL, 8 + 2 * (dst & 3), 0, 0); break;
                    case T_FMUL_R: w0 = wpack(W_FMUL_R, 16 + 2 * (dst & 3), 24 + 2 * (src & 3), 0); break;
                    case T_FDIV_M: w0 = wpack(W_FDIV_M, 16 + 2 * (dst & 3), src, bits12); break;
                    case T_FSQRT_R: w0 = wpack(W_FSQRT, 16 + 2 * (dst & 3), 0, 0); break;
                    case T_CBRANCH: {
                        const u32 shift = (mod >> 4) + 8;
                        w0 = (u32)(usage[dst][t] + 1) | (W_CBRANCH << 8) | (shift << 16) | ((dst * 8) << 24);   // src field = target + 1 (not scaled)
                        w1 = (imm | (1u << shift)) & ~(1u << (shift - 1));
#pragma unroll
                        for (int r = 0; r < 8; r++) usage[r][t] = (short)i;
                    } break;
                    case T_CFROUND: w0 = wpack(W_CFROUND, 0, src, imm & 63); break;
                    case T_ISTORE: w0 = wpack(W_ISTORE, dst, src, (mod >> 4) < 14 ? bits12 : 21); break;
                    default: break;
                }
                b.program[(size_t)vm * kProgramSize + i] = make_uint2(w0, w1);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- the VM
// more than kRcpSlots IMUL_RCP in one program (never observed): kept out of line so its loop does not take registers
// (uniform ones included) away from the interpreter loop
__device__ __noinline__ u64 reciprocal_slow(u32 divisor) { return device_reciprocal(divisor); }
// The rounding mode (fprc) is folded into the interpreter's jump-table index, so every FP handler exists once per
// mode with the mode a compile-time constant: native directed-rounding DADD/DMUL, no branch on the mode.
template <int M> __device__ __forceinline__ double add_c(double a, double c) {
    return M == 0 ? __dadd_rn(a, c) : M == 1 ? __dadd_rd(a, c) : M == 2 ? __dadd_ru(a, c) : __dadd_rz(a, c);
}
template <int M> __device__ __forceinline__ double mul_c(double a, double c) {
    return M == 0 ? __dmul_rn(a, c) : M == 1 ? __dmul_rd(a, c) : M == 2 ? __dmul_ru(a, c) : __dmul_rz(a, c);
}
// e-group values are positive and finite (spec §4.3.2): directed rounding = round-to-nearest, then step one ulp against
// the sign of the exact residual.  residual = fma(-q, b, a) is exact for a correctly rounded quotient / root.
// FDIV_M / FSQRT_R keep the mode a run-time value: their slow paths are large and they are 10 of 256 instructions;
// four copies of them would push the interpreter past the 32 KB instruction cache
__device__ __forceinline__ double fix_positive_rt(double q, double residual, u32 mode) {
    long long bits = __double_as_longlong(q);
    const bool down = (mode == 1 || mode == 3) && residual < 0.0, up = mode == 2 && residual > 0.0;
    bits += up ? 1 : 0;
    bits -= down ? 1 : 0;
    return __longlong_as_double(bits);
}
__device__ __forceinline__ double div_rt(double a, double c, u32 mode) { const double q = __ddiv_rn(a, c); return fix_positive_rt(q, __fma_rn(-q, c, a), mode); }
__device__ __forceinline__ double sqrt_rt(double a, u32 mode) { const double r = __dsqrt_rn(a); return fix_positive_rt(r, __fma_rn(-r, r, a), mode); }
__device__ __forceinline__ u64 d2u(double v) { return (u64)__double_as_longlong(v); }
__device__ __forceinline__ double u2d(u64 v) { return __longlong_as_double((long long)v); }

// ---------------------------------------------------------------------------------------------- the VM: one WARP per VM
// All 32 lanes run the same VM, so the interpreter never diverges: a step costs its own latency, not the worst latency
// among 32 unrelated programs, so a hash finishes soon enough for the verifier's pow check, in 1/8 of the memory.
// Rejected alternatives: one THREAD per VM (register files in shared memory, switch diverging over 32 programs, 8x the
// scratchpads per SM and a batch as slow as its slowest program); a first warp-per-VM kernel with the register file
// spread over the lanes (operands by shuffle, over twice the SASS instructions per VM instruction).  This kernel: the register file lives in shared
// memory (one LDS.64 per operand instead of two shuffles and a convergence check), slot fields of the instruction
// word are byte offsets, opcodes are dense with one opcode per (operation, operand kind) so a handler touches only
// what it needs, and every lane executes the whole instruction redundantly (both halves of an FP register too): no
// cross-lane dependency inside the program loop, no warp synchronisation; the lanes split up only for the 64-byte
// scratchpad / dataset lines around it.  The dispatch is a jump table indexed by opcode | rounding mode, both operands
// are requested before the branch and lane 0 interprets alone; 25 SASS instructions per VM instruction and 23 KB of code — the 32 KB instruction
// cache is a hard budget for an interpreter: a 58 KB build with 30 % fewer instructions per step was slower.
__device__ __forceinline__ uint8_t *sp_byte(uint8_t *cold, uint8_t *hot, u32 addr) { return (addr < kScratchpadL1 ? hot : cold) + addr; }

// Per-warp shared state of the VM kernel.  The interpreter addresses it with explicit 32-bit shared-window addresses
// kept in ordinary registers (ld.shared / st.shared below): left to itself the compiler re-derives the window base
// (S2R CgaCtaId + 2 more) in every handler once the program loop has a jump table in it.  regs is 256-byte aligned so
// "(word & 0xf8) | base" is the source operand's address in one LOP3; everything else is base + constant + field.
template <int WARPS>
struct alignas(256) VmWarpShared {
    u64 regs[32];
    u64 rcp[kRcpSlots];
    u64 emask[2];                      // e-register exponent masks (lo, hi): read by the loop prologue and FDIV_M only
    u32 self[2];                       // shared-window address of regs, read back through a volatile load (see vm_run)
    uint2 prog[kProgramSize + 1];      // + W_END
};
template <int WARPS>
struct VmShared { VmWarpShared<WARPS> w[WARPS]; };

__device__ __forceinline__ u64 lds64(u32 a) { u64 v; asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ uint2 lds64v2(u32 a) { uint2 v; asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ void lds128(u32 a, u64 &lo, u64 &hi) { asm volatile("ld.shared.v2.u64 {%0, %1}, [%2];" : "=l"(lo), "=l"(hi) : "r"(a) : "memory"); }
__device__ __forceinline__ void sts128(u32 a, u64 lo, u64 hi) { asm volatile("st.shared.v2.u64 [%0], {%1, %2};" ::"r"(a), "l"(lo), "l"(hi) : "memory"); }
__device__ __forceinline__ void sts64(u32 a, u64 v) { asm volatile("st.shared.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }

template <int WARPS>
__device__ __forceinline__ void vm_run(VmWarpShared<WARPS> &sh, const BatchBuffers &b, u32 vm, u32 lane, const uint8_t *__restrict__ dataset) {
    uint2 *prog = sh.prog;
    u64 *rcp = sh.rcp, *regs = sh.regs;
    const u64 *emask = sh.emask;
    for (int i = lane; i < kProgramSize; i += 32) prog[i] = b.program[(size_t)vm * kProgramSize + i];
    if (lane == 0) prog[kProgramSize] = make_uint2((u32)W_END << 8, 0);
    rcp[lane] = b.rcp[(size_t)vm * kRcpSlots + lane];
    const u32 stride = b.stride;
    regs[lane] = lane >= 24 ? b.regfile[(size_t)lane * stride + vm] : 0;
    __syncwarp();
    const u64 c0 = b.config[vm], c1 = b.config[(size_t)stride + vm];
    if (lane < 2) sh.emask[lane] = b.config[(size_t)(2 + lane) * stride + vm];
    __syncwarp();
    u32 ma = (u32)c0, mx = (u32)(c0 >> 32);
    const u32 rr = (u32)(c1 >> 60);
    const uint8_t *ds = dataset + (c1 & ((1ull << 60) - 1));
    u32 mode = (u32)b.fprc[vm] << 6;                        // kept pre-shifted: it is OR-ed into the jump-table index
    uint8_t *sp = b.scratchpads + (size_t)vm * kScratchpadL3;
    uint8_t *sph = b.hot + (size_t)vm * kScratchpadL1;      // offsets below 16 KiB (75 % of the accesses) go to the hot plane
    constexpr u64 kEMant = (1ull << 56) - 1;
    // the window address of regs, laundered through shared memory: ptxas sees through a mov and re-derives base + offset
    // inside the loop; it cannot see through a volatile load
    if (lane == 0) sh.self[0] = (u32)__cvta_generic_to_shared(regs);
    __syncwarp();
    const u32 rbase = *reinterpret_cast<volatile u32 *>(&sh.self[0]);
    constexpr u32 kRcpOff = offsetof(VmWarpShared<WARPS>, rcp), kEmaskOff = offsetof(VmWarpShared<WARPS>, emask),
                  kProgOff = offsetof(VmWarpShared<WARPS>, prog);
#define RDA(addr) lds64(addr)
#define WRA(addr, v) sts64((addr), (v))
#define SPTR(addr) sp_byte(sp, sph, (addr))
#define SPAD(addr) (*reinterpret_cast<u64 *>(SPTR(addr)))

    u32 sp0 = mx, sp1 = ma;
    for (int it = 0; it < kProgramIterations; it++) {
        const u64 mix = regs[rr & 1] ^ regs[2 + ((rr >> 1) & 1)];
        sp0 = (sp0 ^ (u32)mix) & kL3Mask64;
        sp1 = (sp1 ^ (u32)(mix >> 32)) & kL3Mask64;
        __syncwarp();                                    // everyone has read `mix` before lanes overwrite their slots
        if (lane < 8) regs[lane] ^= SPAD(sp0 + 8 * lane);
        else if (lane < 24) {
            const int x = *reinterpret_cast<const int *>(SPTR(sp1 + 4 * (lane - 8)));
            const u64 bits = d2u((double)x);
            regs[lane] = lane >= 16 ? ((bits & kEMant) | emask[lane & 1]) : bits;
        }
        __syncwarp();

        // The program is interpreted by lane 0 ALONE (the other lanes wait at the reconvergence point below): every lane
        // would compute the same values, but 32 same-address 64-bit stores cost 2-4 shared-memory wavefronts each and kept
        // the LSU data pipe 72 % busy (ncu) — the resource that flattened throughput beyond 40 VMs per SM.  One active
        // lane: one wavefront per access, same issue cost.
        if (lane == 0) for (u32 pc = rbase + kProgOff;;) {
            const uint2 ins = lds64v2(pc);
            pc += 8;
            const u32 w = ins.x;
            const u32 da = rbase + (w >> 24), sa = (w & 0xf8u) | rbase, aux = __byte_perm(w, 0, 0x4442);   // LEA.HI, LOP3, PRMT
            const u64 simm = sext(ins.y);
            const u64 dv = lds64(da), sv = lds64(sa);        // both operands are requested before the jump-table load and the
                                                             // branch: a handler starts with them in flight (slot fields are valid for every opcode)
#define MEMADDR (((u32)sv + ins.y) & ((1u << aux) - 8u))
#define FP_M(lo, hi) const u64 mv_ = SPAD(MEMADDR); const double lo = (double)(int)(u32)mv_, hi = (double)(int)(u32)(mv_ >> 32)
#define ANY_MODE(op) case op: case op + 64: case op + 128: case op + 192
#define PER_MODE(op, ...) \
    case op: { constexpr int M = 0; __VA_ARGS__ } break; \
    case op + 64: { constexpr int M = 1; __VA_ARGS__ } break; \
    case op + 128: { constexpr int M = 2; __VA_ARGS__ } break; \
    case op + 192: { constexpr int M = 3; __VA_ARGS__ } break;
#define FP_LOAD_D const double dlo = u2d(dv), dhi = u2d(RDA(da + 8))
#define FP_LOAD_S const double slo = u2d(sv), shi = u2d(RDA(sa + 8))
            static_assert(W_COUNT <= 64, "the opcode shares the jump-table index with the rounding mode");
            switch (((w >> 8) & 63) | mode) {
                ANY_MODE(W_IADD_RS): WRA(da, dv + (sv << aux) + simm); break;
                ANY_MODE(W_ISUB_R): WRA(da, dv - sv); break;
                ANY_MODE(W_IMUL_R): WRA(da, dv * sv); break;
                ANY_MODE(W_IMULH_R): WRA(da, mulh_u(dv, sv)); break;
                ANY_MODE(W_ISMULH_R): WRA(da, mulh_s(dv, sv)); break;
                ANY_MODE(W_IXOR_R): WRA(da, dv ^ sv); break;
                ANY_MODE(W_IROR_R): { const u64 d = dv; const u32 c = (u32)sv & 63; WRA(da, (d >> c) | (d << ((64 - c) & 63))); } break;
                ANY_MODE(W_IROL_R): { const u64 d = dv; const u32 c = (u32)sv & 63; WRA(da, (d << c) | (d >> ((64 - c) & 63))); } break;
                ANY_MODE(W_ISWAP): { const u64 d = dv, s = sv; WRA(da, s); WRA(sa, d); } break;
                ANY_MODE(W_ISUB_I): WRA(da, dv - simm); break;
                ANY_MODE(W_IMUL_I): WRA(da, dv * simm); break;
                ANY_MODE(W_IXOR_I): WRA(da, dv ^ simm); break;
                ANY_MODE(W_IROR_I): { const u64 d = dv; WRA(da, (d >> aux) | (d << ((64 - aux) & 63))); } break;
                ANY_MODE(W_IROL_I): { const u64 d = dv; WRA(da, (d << aux) | (d >> ((64 - aux) & 63))); } break;
                ANY_MODE(W_INEG): WRA(da, 0 - dv); break;
                ANY_MODE(W_IMUL_RCP): WRA(da, dv * RDA(rbase + kRcpOff + aux * 8)); break;
                ANY_MODE(W_IMUL_RCP_SLOW): WRA(da, dv * reciprocal_slow(ins.y)); break;
                ANY_MODE(W_IADD_M): WRA(da, dv + SPAD(MEMADDR)); break;
                ANY_MODE(W_ISUB_M): WRA(da, dv - SPAD(MEMADDR)); break;
                ANY_MODE(W_IMUL_M): WRA(da, dv * SPAD(MEMADDR)); break;
                ANY_MODE(W_IMULH_M): WRA(da, mulh_u(dv, SPAD(MEMADDR))); break;
                ANY_MODE(W_ISMULH_M): WRA(da, mulh_s(dv, SPAD(MEMADDR))); break;
                ANY_MODE(W_IXOR_M): WRA(da, dv ^ SPAD(MEMADDR)); break;
                ANY_MODE(W_IADD_A): WRA(da, dv + SPAD(ins.y)); break;
                ANY_MODE(W_ISUB_A): WRA(da, dv - SPAD(ins.y)); break;
                ANY_MODE(W_IMUL_A): WRA(da, dv * SPAD(ins.y)); break;
                ANY_MODE(W_IMULH_A): WRA(da, mulh_u(dv, SPAD(ins.y))); break;
                ANY_MODE(W_ISMULH_A): WRA(da, mulh_s(dv, SPAD(ins.y))); break;
                ANY_MODE(W_IXOR_A): WRA(da, dv ^ SPAD(ins.y)); break;
                ANY_MODE(W_CBRANCH): {
                    const u64 r0 = dv + simm;
                    WRA(da, r0);
                    if ((r0 & (255ull << aux)) == 0) pc = rbase + kProgOff + (w & 255u) * 8;       // low byte = target + 1
                } break;
                ANY_MODE(W_CFROUND): { const u64 s = sv; mode = ((u32)((s >> aux) | (s << ((64 - aux) & 63))) & 3) << 6; } break;
                ANY_MODE(W_ISTORE): SPAD(((u32)dv + ins.y) & ((1u << aux) - 8u)) = sv; break;
                ANY_MODE(W_FSWAP): sts128(da, RDA(da + 8), dv); break;
                ANY_MODE(W_FSCAL): sts128(da, dv ^ 0x80F0000000000000ull, RDA(da + 8) ^ 0x80F0000000000000ull); break;
                PER_MODE(W_FADD_R, FP_LOAD_D; FP_LOAD_S; sts128(da, d2u(add_c<M>(dlo, slo)), d2u(add_c<M>(dhi, shi)));)
                PER_MODE(W_FSUB_R, FP_LOAD_D; FP_LOAD_S; sts128(da, d2u(add_c<M>(dlo, -slo)), d2u(add_c<M>(dhi, -shi)));)
                PER_MODE(W_FMUL_R, FP_LOAD_D; FP_LOAD_S; sts128(da, d2u(mul_c<M>(dlo, slo)), d2u(mul_c<M>(dhi, shi)));)
                ANY_MODE(W_FSQRT): { FP_LOAD_D; const u32 m = mode >> 6; sts128(da, d2u(sqrt_rt(dlo, m)), d2u(sqrt_rt(dhi, m))); } break;
                PER_MODE(W_FADD_M, FP_M(mlo, mhi); FP_LOAD_D; sts128(da, d2u(add_c<M>(dlo, mlo)), d2u(add_c<M>(dhi, mhi)));)
                PER_MODE(W_FSUB_M, FP_M(mlo, mhi); FP_LOAD_D; sts128(da, d2u(add_c<M>(dlo, -mlo)), d2u(add_c<M>(dhi, -mhi)));)
                ANY_MODE(W_FDIV_M): { FP_M(mlo, mhi); FP_LOAD_D; u64 el, eh; lds128(rbase + kEmaskOff, el, eh);
                         const double vlo = u2d((d2u(mlo) & kEMant) | el), vhi = u2d((d2u(mhi) & kEMant) | eh);
                         const u32 m = mode >> 6; sts128(da, d2u(div_rt(dlo, vlo, m)), d2u(div_rt(dhi, vhi, m))); } break;
                ANY_MODE(W_NOP): break;
                ANY_MODE(W_END): goto program_done;
                default: __builtin_unreachable();     // the decoder emits nothing else: lets the jump table drop its range check
            }
#undef ANY_MODE
#undef PER_MODE
#undef FP_LOAD_D
#undef FP_LOAD_S
#undef MEMADDR
#undef FP_M
        }
    program_done:
        __syncwarp();
        mode = __shfl_sync(0xffffffffu, mode, 0);

        mx = (mx ^ (u32)(regs[4 + ((rr >> 2) & 1)] ^ regs[6 + ((rr >> 3) & 1)])) & kDatasetAlignMask;
        if (lane == 0) asm volatile("prefetch.global.L2 [%0];" ::"l"(ds + mx));
        __syncwarp();                                    // program-loop writes (all lanes, same values) settle before the lanes split
        if (lane < 8) {
            const u64 v = regs[lane] ^ __ldg(reinterpret_cast<const u64 *>(ds + ma) + lane);
            regs[lane] = v;
            SPAD(sp1 + 8 * lane) = v;
        } else if (lane < 16) {
            const u64 v = regs[lane] ^ regs[lane + 8];
            regs[lane] = v;                              // f ^= e; written after the r line: the two may share a scratchpad line
        }
        { const u32 tmp = mx; mx = ma; ma = tmp; }
        __syncwarp();
        if (lane >= 8 && lane < 16) SPAD(sp0 + 8 * (lane - 8)) = regs[lane];
        __syncwarp();
        sp0 = 0; sp1 = 0;
    }
    if (lane < 24) b.regfile[(size_t)lane * stride + vm] = regs[lane];
    if (lane == 0) b.fprc[vm] = (uint8_t)(mode >> 6);
#undef RDA
#undef WRA
#undef SPAD
#undef SPTR
}

template <int WARPS, int MIN_CTAS>
__global__ void __launch_bounds__(WARPS * 32, MIN_CTAS) execute_kernel(BatchBuffers b, u32 n, const uint8_t *__restrict__ dataset) {
    __shared__ VmShared<WARPS> sh;
    const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5, vm = blockIdx.x * WARPS + wid;
    if (vm >= n) return;
    vm_run<WARPS>(sh.w[wid], b, vm, lane, dataset);
}

// ---------------------------------------------------------------------------------------------- chain seed / final hash
__global__ void chain_seed_kernel(BatchBuffers b, u32 n, bool final_hash) {
    const u32 vm = blockIdx.x * blockDim.x + threadIdx.x;
    if (vm >= n) return;
    u64 h[8], m[16];
    b2_init(h, final_hash ? 32 : 64);
    for (int i = 0; i < 16; i++) m[i] = b.regfile[(size_t)i * b.stride + vm];
    b2_compress(h, m, 128, false);
    for (int i = 0; i < 16; i++) m[i] = b.regfile[(size_t)(16 + i) * b.stride + vm];
    b2_compress(h, m, 256, true);
    if (final_hash) { u64 *out = reinterpret_cast<u64 *>(b.hashes + (size_t)vm * 32); for (int i = 0; i < 4; i++) out[i] = h[i]; }
    else for (int i = 0; i < 8; i++) b.seed[(size_t)i * b.stride + vm] = h[i];
}

__global__ void find_below_kernel(const uint8_t *__restrict__ hashes, u32 n, const uint8_t *__restrict__ difficulty, u32 *found) {
    const u32 vm = blockIdx.x * blockDim.x + threadIdx.x;
    if (vm >= n) return;
    const uint8_t *h = hashes + (size_t)vm * 32;
    for (int i = 0; i < 32; i++) {               // big-endian byte order: the first differing byte decides
        const uint8_t a = h[i], d = difficulty[i];
        if (a != d) { if (a < d) atomicMin(found, vm); return; }
    }
}

inline u32 blocks_for(u64 n, u32 per) { return (u32)((n + per - 1) / per); }

}  // namespace

// ------------------------------------------------------------------------------------------------ host-side launchers
cudaError_t upload_tables() {
    // AES: S-box from the field inverse + affine map (FIPS-197 §5.1.1), then the MixColumns-folded round tables
    uint8_t sbox[256], inv[256];
    auto xt = [](uint8_t a) { return (uint8_t)((a << 1) ^ ((a & 0x80) ? 0x1b : 0)); };
    auto gm = [&](uint8_t a, uint8_t c) { uint8_t p = 0; for (int i = 0; i < 8; i++) { if (c & 1) p ^= a; a = xt(a); c >>= 1; } return p; };
    uint8_t ex[256], lg[256], x = 1;
    for (int i = 0; i < 255; i++) { ex[i] = x; lg[x] = (uint8_t)i; x = (uint8_t)(x ^ xt(x)); }
    for (int v = 0; v < 256; v++) {
        const uint8_t iv = v ? ex[(255 - lg[v]) % 255] : 0;
        uint8_t s = iv, r = iv;
        for (int k = 0; k < 4; k++) { r = (uint8_t)((r << 1) | (r >> 7)); s ^= r; }
        sbox[v] = s ^ 0x63;
    }
    for (int v = 0; v < 256; v++) inv[sbox[v]] = (uint8_t)v;
    u32 te[256], td[256];
    for (int v = 0; v < 256; v++) {
        const uint8_t s = sbox[v], i = inv[v];
        te[v] = (u32)gm(s, 2) | ((u32)s << 8) | ((u32)s << 16) | ((u32)gm(s, 3) << 24);
        td[v] = (u32)gm(i, 14) | ((u32)gm(i, 9) << 8) | ((u32)gm(i, 13) << 16) | ((u32)gm(i, 11) << 24);
    }
    cudaError_t e;
    if ((e = cudaMemcpyToSymbol(g_te0, te, sizeof te)) != cudaSuccess) return e;
    if ((e = cudaMemcpyToSymbol(g_td0, td, sizeof td)) != cudaSuccess) return e;
    static const uint8_t freq[T_COUNT] = {16, 7, 16, 7, 16, 4, 4, 1, 4, 1, 8, 2, 15, 5, 8, 2, 4, 4, 16, 5, 16, 5, 6, 32, 4, 6, 25, 1, 16, 0};
    uint8_t opmap[256]; int k = 0;
    for (int t = 0; t < T_COUNT; t++) for (int j = 0; j < freq[t]; j++) opmap[k++] = (uint8_t)t;
    if ((e = cudaMemcpyToSymbol(g_opmap, opmap, sizeof opmap)) != cudaSuccess) return e;
    uint8_t g1[64], g4[128], hs[64], hx[32];
    blake2b(g1, 64, "RandomX AesGenerator1R keys", 27);
    blake2b(g4, 64, "RandomX AesGenerator4R keys 0-3", 31);
    blake2b(g4 + 64, 64, "RandomX AesGenerator4R keys 4-7", 31);
    blake2b(hs, 64, "RandomX AesHash1R state", 23);
    blake2b(hx, 32, "RandomX AesHash1R xkeys", 23);
    if ((e = cudaMemcpyToSymbol(c_gen1_keys, g1, 64)) != cudaSuccess) return e;
    if ((e = cudaMemcpyToSymbol(c_gen4_keys, g4, 128)) != cudaSuccess) return e;
    if ((e = cudaMemcpyToSymbol(c_hash_state, hs, 64)) != cudaSuccess) return e;
    return cudaMemcpyToSymbol(c_hash_xkeys, hx, 32);
}

cudaError_t launch_dataset(const uint64_t *d_cache, const SuperscalarImage &ss, uint64_t *d_dataset, uint64_t first, uint64_t count, cudaStream_t s) {
    SsArgs a;
    a.ops = ss.ops;
    memcpy(a.first, ss.first, sizeof a.first);
    memcpy(a.address_reg, ss.address_reg, sizeof a.address_reg);
    dataset_kernel<<<blocks_for(count, kDatasetThreads), kDatasetThreads, 0, s>>>(reinterpret_cast<const u64 *>(d_cache), a, reinterpret_cast<u64 *>(d_dataset), first, count);
    return cudaGetLastError();
}
cudaError_t launch_seed_inputs(const BatchBuffers &b, uint32_t n, const uint8_t *d_inputs, uint32_t input_len, cudaStream_t s) {
    seed_inputs_kernel<<<blocks_for(n, 128), 128, 0, s>>>(reinterpret_cast<u64 *>(b.seed), b.stride, n, d_inputs, input_len);
    return cudaGetLastError();
}
cudaError_t launch_seed_k2pow(const BatchBuffers &b, uint32_t n, const K2powTemplate &t, cudaStream_t s) {
    seed_k2pow_kernel<<<blocks_for(n, 128), 128, 0, s>>>(reinterpret_cast<u64 *>(b.seed), b.stride, n, t);
    return cudaGetLastError();
}
cudaError_t launch_fill_scratchpads(const BatchBuffers &b, uint32_t n, cudaStream_t s) {
    fill_kernel<<<blocks_for((u64)n * 4, 256), 256, 0, s>>>(reinterpret_cast<u64 *>(b.seed), b.stride, n, b.scratchpads, b.hot);
    return cudaGetLastError();
}
cudaError_t launch_program(const BatchBuffers &b, uint32_t n, bool first_program, cudaStream_t s) {
    program_kernel<<<blocks_for(n, 128), 128, 0, s>>>(b, n, first_program);
    return cudaGetLastError();
}
cudaError_t launch_execute(const BatchBuffers &b, uint32_t n, const uint64_t *d_dataset, int variant, cudaStream_t s) {
    const uint8_t *ds = reinterpret_cast<const uint8_t *>(d_dataset);
    switch (variant) {
        case 1: execute_kernel<2, 24><<<blocks_for(n, 2), 64, 0, s>>>(b, n, ds); break;    // <= 42 registers: 48 warps per SM
        case 2: execute_kernel<2, 32><<<blocks_for(n, 2), 64, 0, s>>>(b, n, ds); break;    // <= 32 registers: 64 warps per SM
        case 3: execute_kernel<2, 20><<<blocks_for(n, 2), 64, 0, s>>>(b, n, ds); break;    // <= 51 registers: 40 warps per SM
        default: execute_kernel<1, 32><<<n, 32, 0, s>>>(b, n, ds); break;                  // <= 64 registers: 32 warps per SM
    }
    return cudaGetLastError();
}
cudaError_t launch_chain_seed(const BatchBuffers &b, uint32_t n, cudaStream_t s) {
    chain_seed_kernel<<<blocks_for(n, 128), 128, 0, s>>>(b, n, false);
    return cudaGetLastError();
}
cudaError_t launch_finalize(const BatchBuffers &b, uint32_t n, cudaStream_t s) {
    hash_scratchpad_kernel<<<blocks_for((u64)n * 4, 256), 256, 0, s>>>(reinterpret_cast<u64 *>(b.regfile), b.stride, n, b.scratchpads, b.hot);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    chain_seed_kernel<<<blocks_for(n, 128), 128, 0, s>>>(b, n, true);
    return cudaGetLastError();
}
cudaError_t launch_find_below(const BatchBuffers &b, uint32_t n, const uint8_t *d_difficulty, uint32_t *d_found, cudaStream_t s) {
    find_below_kernel<<<blocks_for(n, 256), 256, 0, s>>>(b.hashes, n, d_difficulty, d_found);
    return cudaGetLastError();
}

}  // namespace rx
}  // namespace b200post
