// label_sums.h — block digests of POST labels (DESIGN.md §3g): the BLAKE3 kernel's host side, and the digests of one
// file built from its labels in order, which the setup sessions and b200post_write_sums save as postdata_<N>.sum.
#pragma once
#include <cstdint>
#include <string>

#include "cuda_util.h"
#include "postdata_io.h"

namespace b200post {

// BLAKE3 digests of label blocks on one device (the kernel of label_sums.cu)
class BlockHasher {
public:
    explicit BlockHasher(int device) : dev_(device) {}
    BlockHasher(const BlockHasher &) = delete;
    // `count` labels in host memory (pinned or not), split into blocks of kSumBlockLabels from the first, the last one
    // possibly short: one 32-byte digest per block into out.  Returns once the digests are in out.
    int digests(const uint8_t *labels, uint64_t count, uint8_t *out);
    int device() const { return dev_; }

private:
    int dev_;
    Stream stream_;
    DeviceBuffer<uint8_t> d_in_, d_out_;
};

// One digest range of a chunk already in device memory: `bytes` (a positive multiple of 16, at most 1 MiB) from byte
// `offset` of the chunk
struct DigestDesc { uint64_t offset; uint32_t bytes, pad; };
// Enqueues on `st` the digests of the n ranges d_desc[0, n) (device) of the chunk at d_chunk, one CTA each: range i's
// digest into d_out[32 i, 32 i + 32).  The proving scan's check of each chunk against its sidecars.
cudaError_t launch_range_digests(cudaStream_t st, const uint8_t *d_chunk, const DigestDesc *d_desc, uint32_t n, uint8_t *d_out);

// The sidecar of one file under construction: feed() takes the file's labels in order from sums().covered on, hashes
// every block they complete, and keeps the bytes of a block they leave open; save() hashes that open block as the
// sidecar's short last one and writes the file.  The bytes fed are hashed, never read back from disk.
class FileSums {
public:
    // keeps the whole blocks of `from` (absent = none) below `keep`, a multiple of kSumBlockLabels
    FileSums(const PostSums &from, uint64_t keep);
    uint64_t covered() const { return full_ * kSumBlockLabels + open_.size() / 16; }
    uint64_t file() const { return sums_.file; }
    // labels [covered(), covered() + n); *completed (may be NULL) says whether they completed a block
    int feed(BlockHasher &h, const uint8_t *labels, uint64_t n, bool *completed = nullptr);
    int save(BlockHasher &h, const std::string &dir);
    // the sidecar as save() writes it
    int sums(BlockHasher &h, PostSums *out);

private:
    PostSums sums_;          // header, and the digests of the whole blocks
    uint64_t full_ = 0;      // whole blocks hashed
    std::string open_;       // bytes of the open block
};

}  // namespace b200post
