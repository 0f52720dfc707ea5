// label_sums.cu — BLAKE3 digests of 1 MiB blocks of POST labels (DESIGN.md §3g), the block checksums that
// postdata_<N>.sum stores, and their host side (label_sums.h).
//
// A block's digest is unkeyed BLAKE3 of its bytes, 32-byte output.  One CTA hashes one block: each thread runs the
// 16 compressions of one 1 KiB chunk at a time (CHUNK_START / CHUNK_END, chunk counter = chunk index in the block),
// writes the chunk's chaining value to shared memory, and the parent levels are reduced there.  Merging neighbours
// pairwise and carrying an odd last node up a level builds BLAKE3's tree for any chunk count (the left subtree is
// always the largest power of two of chunks), and the top node is compressed with ROOT.  A short block may end in a
// partial chunk and a partial 64-byte message block; a one-chunk block is its own root.
#include <algorithm>
#include <cstring>

#include "../../include/b200post_setup.h"
#include "engine.h"
#include "label_sums.h"

namespace b200post {
namespace {

constexpr uint32_t kChunkBytes = 1024;
constexpr uint32_t kBlockBytes = (uint32_t)kSumBlockLabels * 16;
constexpr uint32_t kMaxChunks = kBlockBytes / kChunkBytes;   // 1024
constexpr int kSumThreads = 256;
constexpr uint64_t kMaxLaunchBlocks = 64;                    // 64 MiB of labels per launch
enum : uint32_t { CHUNK_START = 1, CHUNK_END = 2, PARENT = 4, ROOT = 8 };

__device__ __forceinline__ uint32_t rotr(uint32_t x, int n) { return __funnelshift_r(x, x, n); }

#define B3_G(a, b, c, d, x, y)                                                 \
    a = a + b + x; d = rotr(d ^ a, 16); c = c + d; b = rotr(b ^ c, 12);        \
    a = a + b + y; d = rotr(d ^ a, 8); c = c + d; b = rotr(b ^ c, 7);

// cv <- the first 8 words of compress(cv, m, counter, len, flags)
__device__ __forceinline__ void compress(uint32_t cv[8], const uint32_t min[16], uint64_t counter, uint32_t len, uint32_t flags) {
    uint32_t v[16] = {cv[0], cv[1], cv[2], cv[3], cv[4], cv[5], cv[6], cv[7], 0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au,
                      (uint32_t)counter, (uint32_t)(counter >> 32), len, flags};
    uint32_t m[16];
#pragma unroll
    for (int i = 0; i < 16; i++) m[i] = min[i];
#pragma unroll
    for (int r = 0; r < 7; r++) {
        B3_G(v[0], v[4], v[8], v[12], m[0], m[1]);
        B3_G(v[1], v[5], v[9], v[13], m[2], m[3]);
        B3_G(v[2], v[6], v[10], v[14], m[4], m[5]);
        B3_G(v[3], v[7], v[11], v[15], m[6], m[7]);
        B3_G(v[0], v[5], v[10], v[15], m[8], m[9]);
        B3_G(v[1], v[6], v[11], v[12], m[10], m[11]);
        B3_G(v[2], v[7], v[8], v[13], m[12], m[13]);
        B3_G(v[3], v[4], v[9], v[14], m[14], m[15]);
        if (r < 6) {   // BLAKE3's message permutation; with the loop unrolled it is a renaming of registers
            const uint32_t t[16] = {m[2], m[6], m[3], m[10], m[7], m[0], m[4], m[13], m[1], m[11], m[12], m[5], m[9], m[14], m[15], m[8]};
#pragma unroll
            for (int i = 0; i < 16; i++) m[i] = t[i];
        }
    }
#pragma unroll
    for (int i = 0; i < 8; i++) cv[i] = v[i] ^ v[i + 8];
}

__device__ __forceinline__ void load_iv(uint32_t cv[8]) {
    cv[0] = 0x6A09E667u; cv[1] = 0xBB67AE85u; cv[2] = 0x3C6EF372u; cv[3] = 0xA54FF53Au;
    cv[4] = 0x510E527Fu; cv[5] = 0x9B05688Cu; cv[6] = 0x1F83D9ABu; cv[7] = 0x5BE0CD19u;
}

// The digest of one block of `bytes` (a positive multiple of 16, at most kBlockBytes) at base, by the whole CTA, into
// out[0, 32).  Shared by the kernel over host-copied blocks and the one over ranges of a device-resident chunk.
__device__ __forceinline__ void hash_block(const uint8_t *__restrict__ base, uint32_t bytes, uint8_t *__restrict__ out) {
    __shared__ uint32_t cvs[kMaxChunks][8];
    const uint32_t n_chunks = (bytes + kChunkBytes - 1) / kChunkBytes;
    const uint32_t root_chunk = n_chunks == 1 ? ROOT : 0;

    for (uint32_t c = threadIdx.x; c < n_chunks; c += kSumThreads) {
        const uint32_t cb = min(kChunkBytes, bytes - c * kChunkBytes);
        const uint32_t n_msg = (cb + 63) / 64;
        uint32_t cv[8];
        load_iv(cv);
        for (uint32_t j = 0; j < n_msg; j++) {
            const uint32_t len = min(64u, cb - j * 64);
            const uint4 *p = reinterpret_cast<const uint4 *>(base + (size_t)c * kChunkBytes + j * 64);
            uint32_t m[16];
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const uint4 w = q * 16 < (int)len ? __ldg(p + q) : make_uint4(0, 0, 0, 0);
                m[4 * q] = w.x; m[4 * q + 1] = w.y; m[4 * q + 2] = w.z; m[4 * q + 3] = w.w;
            }
            const uint32_t flags = (j == 0 ? CHUNK_START : 0) | (j + 1 == n_msg ? CHUNK_END | root_chunk : 0);
            compress(cv, m, c, len, flags);
        }
#pragma unroll
        for (int i = 0; i < 8; i++) cvs[c][i] = cv[i];
    }
    __syncthreads();

    // parent levels: node i of the next level is parent(2i, 2i + 1); an odd last node moves up unchanged
    for (uint32_t n = n_chunks; n > 1; n = (n + 1) / 2) {
        const uint32_t pairs = n / 2;
        const uint32_t flags = PARENT | (n == 2 ? ROOT : 0);
        uint32_t res[2][8];
#pragma unroll
        for (int k = 0; k < 2; k++) {   // pairs <= kMaxChunks / 2 = 2 x kSumThreads
            const uint32_t i = threadIdx.x + k * kSumThreads;
            if (i < pairs) {
                uint32_t m[16];
#pragma unroll
                for (int w = 0; w < 8; w++) { m[w] = cvs[2 * i][w]; m[8 + w] = cvs[2 * i + 1][w]; }
                load_iv(res[k]);
                compress(res[k], m, 0, 64, flags);
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const uint32_t i = threadIdx.x + k * kSumThreads;
            if (i < pairs) {
#pragma unroll
                for (int w = 0; w < 8; w++) cvs[i][w] = res[k][w];
            }
        }
        if ((n & 1) && threadIdx.x == 0) {
#pragma unroll
            for (int w = 0; w < 8; w++) cvs[pairs][w] = cvs[n - 1][w];
        }
        __syncthreads();
    }
    if (threadIdx.x < 8) reinterpret_cast<uint32_t *>(out)[threadIdx.x] = cvs[0][threadIdx.x];
}

// Blocks [0, full_blocks) of 1 MiB, then, when last_bytes > 0, one short block of last_bytes (a multiple of 16) bytes:
// the digest of block b goes to out[32 b, 32 b + 32).
__global__ void __launch_bounds__(kSumThreads) label_block_digests_kernel(const uint8_t *__restrict__ labels, uint32_t full_blocks,
                                                                          uint32_t last_bytes, uint8_t *__restrict__ out) {
    const uint32_t b = blockIdx.x;
    hash_block(labels + (size_t)b * kBlockBytes, b < full_blocks ? kBlockBytes : last_bytes, out + (size_t)b * 32);
}

// One CTA per range of a chunk already in device memory: range b is desc[b] (byte offset into chunk, bytes), its
// digest goes to out[32 b, 32 b + 32).  The proving scan's digests (b200post_generate_proof_sums).
__global__ void __launch_bounds__(kSumThreads) label_range_digests_kernel(const uint8_t *__restrict__ chunk, const DigestDesc *__restrict__ desc,
                                                                          uint8_t *__restrict__ out) {
    const DigestDesc d = desc[blockIdx.x];
    hash_block(chunk + d.offset, d.bytes, out + (size_t)blockIdx.x * 32);
}

}  // namespace

int BlockHasher::digests(const uint8_t *labels, uint64_t count, uint8_t *out) {
    if (count == 0) return B200POST_OK;
    CUDA_TRY(cudaSetDevice(dev_));
    if (!stream_.get()) CUDA_TRY(stream_.create(cudaStreamNonBlocking));
    const uint64_t blocks = (count + kSumBlockLabels - 1) / kSumBlockLabels;
    const uint64_t per_launch = std::min<uint64_t>(blocks, kMaxLaunchBlocks);
    CUDA_TRY(d_in_.grow((size_t)per_launch * kBlockBytes));
    CUDA_TRY(d_out_.grow((size_t)per_launch * 32));
    for (uint64_t b0 = 0; b0 < blocks; b0 += kMaxLaunchBlocks) {
        const uint64_t first = b0 * kSumBlockLabels, n = std::min<uint64_t>(count - first, kMaxLaunchBlocks * kSumBlockLabels);
        const uint32_t full = (uint32_t)(n / kSumBlockLabels), last_bytes = (uint32_t)(n % kSumBlockLabels * 16);
        const uint32_t grid = full + (last_bytes ? 1 : 0);
        CUDA_TRY(cudaMemcpyAsync(d_in_.get(), labels + first * 16, (size_t)n * 16, cudaMemcpyHostToDevice, stream_.get()));
        label_block_digests_kernel<<<grid, kSumThreads, 0, stream_.get()>>>(d_in_.get(), full, last_bytes, d_out_.get());
        CUDA_TRY(cudaGetLastError());
        g_launches++;
        CUDA_TRY(cudaMemcpyAsync(out + b0 * 32, d_out_.get(), (size_t)grid * 32, cudaMemcpyDeviceToHost, stream_.get()));
        CUDA_TRY(cudaStreamSynchronize(stream_.get()));
    }
    return B200POST_OK;
}

FileSums::FileSums(const PostSums &from, uint64_t keep) : sums_(from) {
    full_ = std::min<uint64_t>(keep, from.covered) / kSumBlockLabels;
    sums_.digests.resize((size_t)full_ * 32);
    sums_.covered = full_ * kSumBlockLabels;
}

int FileSums::feed(BlockHasher &h, const uint8_t *labels, uint64_t n, bool *completed) {
    if (completed) *completed = false;
    if (!open_.empty()) {   // finish the open block first
        const uint64_t take = std::min<uint64_t>(n, kSumBlockLabels - open_.size() / 16);
        open_.append(reinterpret_cast<const char *>(labels), (size_t)take * 16);
        labels += take * 16; n -= take;
        if (open_.size() < kBlockBytes) return B200POST_OK;
        uint8_t d[32];
        if (int rc = h.digests(reinterpret_cast<const uint8_t *>(open_.data()), kSumBlockLabels, d)) return rc;
        sums_.digests.append(reinterpret_cast<const char *>(d), 32);
        full_++; open_.clear();
        if (completed) *completed = true;
    }
    const uint64_t whole = n / kSumBlockLabels;
    if (whole) {
        const size_t at = sums_.digests.size();
        sums_.digests.resize(at + (size_t)whole * 32);
        if (int rc = h.digests(labels, whole * kSumBlockLabels, reinterpret_cast<uint8_t *>(&sums_.digests[at]))) {
            sums_.digests.resize(at);
            return rc;
        }
        full_ += whole;
        if (completed) *completed = true;
    }
    open_.append(reinterpret_cast<const char *>(labels + whole * kSumBlockLabels * 16), (size_t)(n - whole * kSumBlockLabels) * 16);
    return B200POST_OK;
}

int FileSums::sums(BlockHasher &h, PostSums *out) {
    *out = sums_;
    out->digests.resize((size_t)full_ * 32);
    out->covered = covered();
    if (!open_.empty()) {
        uint8_t d[32];
        if (int rc = h.digests(reinterpret_cast<const uint8_t *>(open_.data()), open_.size() / 16, d)) return rc;
        out->digests.append(reinterpret_cast<const char *>(d), 32);
    }
    return B200POST_OK;
}

int FileSums::save(BlockHasher &h, const std::string &dir) {
    PostSums s;
    if (int rc = sums(h, &s)) return rc;
    return save_post_sums(dir, s);
}

cudaError_t launch_range_digests(cudaStream_t st, const uint8_t *d_chunk, const DigestDesc *d_desc, uint32_t n, uint8_t *d_out) {
    if (n == 0) return cudaSuccess;
    label_range_digests_kernel<<<n, kSumThreads, 0, st>>>(d_chunk, d_desc, d_out);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace b200post

using namespace b200post;

extern "C" int b200post_label_block_digests(uint32_t provider, const uint8_t *labels16, uint64_t count, uint8_t *digests32) {
    if ((!labels16 || !digests32) && count) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid argument");
    if (int rc = device_engine(provider)) return rc;
    BlockHasher h((int)provider);
    return h.digests(labels16, count, digests32);
}
