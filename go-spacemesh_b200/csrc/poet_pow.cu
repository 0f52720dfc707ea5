// poet_pow.cu — PoET registration PoW nonce search (include/b200post_poet.h, SURVEY.md §8f.4).
//
// K7 poet_pow_kernel: one SHA-256 compression per candidate nonce from a host-computed midstate; every thread
// walks a strided slice of the chunk and the lowest valid nonce of the chunk is kept with a 64-bit atomicMin.
// Chunks are searched in ascending order, so the first chunk with a hit yields the globally lowest nonce —
// the same answer the reference's sequential loop gives.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b200post_poet.h"
#include "engine.h"
#include "post_device.cuh"

namespace b200post {
namespace {

struct PowJob {
    uint32_t mid[8];        // SHA-256 state after the full 64-byte blocks of the prefix
    uint32_t tail[32];      // remaining prefix bytes + 0x80 padding + bit length, nonce bytes zero (big-endian words)
    uint32_t n_blocks;      // 1 or 2 tail blocks
    uint32_t nonce_word;    // index of the word that receives bswap32(low 32 bits of the nonce)
    uint32_t difficulty;    // required leading zero bits (0..256)
};

__device__ __forceinline__ bool leading_zero_bits_ok(const uint32_t (&st)[8], uint32_t difficulty) {
    uint32_t need = difficulty;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        if (need == 0) return true;
        if (need >= 32) { if (st[i] != 0) return false; need -= 32; }
        else return (st[i] >> (32 - need)) == 0;
    }
    return need == 0;
}

__global__ void __launch_bounds__(256) poet_pow_kernel(const PowJob job, uint64_t first, uint64_t count, unsigned long long *best) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < count; k += stride) {
        const uint64_t nonce = first + k;
        if (nonce >= *(volatile unsigned long long *)best) return;   // a lower valid nonce is known: this thread only goes up
        const uint32_t lo = bswap32((uint32_t)nonce), hi = bswap32((uint32_t)(nonce >> 32));
        uint32_t st[8], w[16];
#pragma unroll
        for (int i = 0; i < 8; i++) st[i] = job.mid[i];
#pragma unroll
        for (int i = 0; i < 16; i++) {
            w[i] = job.tail[i];
            if ((uint32_t)i == job.nonce_word) w[i] = lo;
            if ((uint32_t)i == job.nonce_word + 1) w[i] = hi;
        }
        sha256_compress(st, w);
        if (job.n_blocks == 2) {
#pragma unroll
            for (int i = 0; i < 16; i++) {
                w[i] = job.tail[16 + i];
                if ((uint32_t)(16 + i) == job.nonce_word) w[i] = lo;
                if ((uint32_t)(16 + i) == job.nonce_word + 1) w[i] = hi;
            }
            sha256_compress(st, w);
        }
        if (leading_zero_bits_ok(st, job.difficulty)) atomicMin(best, (unsigned long long)nonce);
    }
}

// host SHA-256 pieces (product-side: the midstate and the one-candidate hash)
void host_compress(uint32_t st[8], const uint8_t block[64]) {
    uint32_t s[8], w[16];
    for (int i = 0; i < 8; i++) s[i] = st[i];
    for (int i = 0; i < 16; i++) w[i] = ((uint32_t)block[4 * i] << 24) | ((uint32_t)block[4 * i + 1] << 16) | ((uint32_t)block[4 * i + 2] << 8) | block[4 * i + 3];
    uint32_t (&sr)[8] = s;
    uint32_t (&wr)[16] = w;
    sha256_compress(sr, wr);
    for (int i = 0; i < 8; i++) st[i] = s[i];
}

// builds prefix || LE64(nonce) with padding; returns false if the layout is unsupported
bool build_job(const uint8_t *pc, size_t pc_len, const uint8_t *ch, size_t ch_len, const uint8_t node_id[32], uint32_t difficulty, PowJob *job,
               std::vector<uint8_t> *message_out = nullptr, uint64_t nonce = 0) {
    std::vector<uint8_t> msg;
    msg.insert(msg.end(), pc, pc + pc_len);
    msg.insert(msg.end(), node_id, node_id + 32);
    msg.insert(msg.end(), ch, ch + ch_len);
    const size_t prefix = msg.size();
    if (prefix % 4) return false;
    for (int i = 0; i < 8; i++) msg.push_back((uint8_t)(nonce >> (8 * i)));
    if (message_out) *message_out = msg;
    const uint64_t bits = (uint64_t)msg.size() * 8;
    msg.push_back(0x80);
    while (msg.size() % 64 != 56) msg.push_back(0);
    for (int i = 7; i >= 0; i--) msg.push_back((uint8_t)(bits >> (8 * i)));
    const size_t full = prefix / 64;   // blocks fully covered by the constant prefix
    uint32_t st[8];
    sha256_iv(st);
    for (size_t b = 0; b < full; b++) host_compress(st, msg.data() + 64 * b);
    const size_t tail_blocks = msg.size() / 64 - full;
    if (tail_blocks < 1 || tail_blocks > 2) return false;
    memset(job, 0, sizeof *job);
    memcpy(job->mid, st, 32);
    for (size_t i = 0; i < tail_blocks * 16; i++) {
        const uint8_t *p = msg.data() + 64 * full + 4 * i;
        job->tail[i] = ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
    }
    job->n_blocks = (uint32_t)tail_blocks;
    job->nonce_word = (uint32_t)((prefix - 64 * full) / 4);
    job->tail[job->nonce_word] = 0; job->tail[job->nonce_word + 1] = 0;
    job->difficulty = difficulty;
    return true;
}

}  // namespace
}  // namespace b200post

using namespace b200post;

extern "C" {

void b200post_poet_pow_hash(const uint8_t *pc, size_t pc_len, const uint8_t *ch, size_t ch_len, const uint8_t node_id[32], uint64_t nonce,
                            uint8_t out[32]) {
    std::vector<uint8_t> msg;
    msg.insert(msg.end(), pc, pc + pc_len);
    msg.insert(msg.end(), node_id, node_id + 32);
    msg.insert(msg.end(), ch, ch + ch_len);
    for (int i = 0; i < 8; i++) msg.push_back((uint8_t)(nonce >> (8 * i)));
    const uint64_t bits = (uint64_t)msg.size() * 8;
    msg.push_back(0x80);
    while (msg.size() % 64 != 56) msg.push_back(0);
    for (int i = 7; i >= 0; i--) msg.push_back((uint8_t)(bits >> (8 * i)));
    uint32_t st[8];
    sha256_iv(st);
    for (size_t b = 0; b < msg.size() / 64; b++) host_compress(st, msg.data() + 64 * b);
    for (int i = 0; i < 8; i++) { out[4 * i] = (uint8_t)(st[i] >> 24); out[4 * i + 1] = (uint8_t)(st[i] >> 16); out[4 * i + 2] = (uint8_t)(st[i] >> 8); out[4 * i + 3] = (uint8_t)st[i]; }
}

int b200post_poet_pow_find(uint32_t provider, const uint8_t *pc, size_t pc_len, const uint8_t *ch, size_t ch_len, const uint8_t node_id[32],
                           uint32_t difficulty, uint64_t start_nonce, uint64_t max_nonces, uint64_t *nonce, uint64_t *hashes,
                           const volatile int *cancel) {
    if ((!pc && pc_len) || (!ch && ch_len) || !node_id || !nonce || difficulty > 256) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    DeviceEngine *e;
    if (int rc = device_engine(provider, &e)) return rc;
    PowJob job;
    if (!build_job(pc, pc_len, ch, ch_len, node_id, difficulty, &job)) {
        set_error("unsupported message layout: challenge lengths must add up to a multiple of 4 bytes");
        return B200POST_ERR_INVALID_ARGUMENT;
    }
    if (cudaSetDevice(e->device()) != cudaSuccess) { set_error("cudaSetDevice failed"); return B200POST_ERR_CUDA; }
    DeviceBuffer<unsigned long long> d_best;
    if (d_best.resize(1) != cudaSuccess) { set_error("cudaMalloc failed"); return B200POST_ERR_CUDA; }
    const uint64_t chunk = 1ull << 28;
    const int grid = e->prop().multiProcessorCount * 8;
    uint64_t done = 0;
    int rc = B200POST_ERR_INVALID_PROOF;
    while (done < max_nonces) {
        if (cancel && *cancel) { rc = B200POST_ERR_CANCELLED; set_error("cancelled"); break; }
        const uint64_t n = std::min<uint64_t>(chunk, max_nonces - done);
        unsigned long long best = ~0ull;
        cudaMemcpy(d_best.get(), &best, 8, cudaMemcpyHostToDevice);
        poet_pow_kernel<<<grid, 256>>>(job, start_nonce + done, n, d_best.get());
        g_launches += 1;
        if (cudaMemcpy(&best, d_best.get(), 8, cudaMemcpyDeviceToHost) != cudaSuccess) { set_error(std::string("poet_pow_kernel: ") + cudaGetErrorString(cudaGetLastError())); rc = B200POST_ERR_CUDA; break; }
        done += n;
        if (best != ~0ull) { *nonce = best; rc = B200POST_OK; break; }
    }
    if (rc == B200POST_ERR_INVALID_PROOF) set_error("no valid nonce in the search window");
    if (hashes) *hashes = done;
    return rc;
}

}  // extern "C"
