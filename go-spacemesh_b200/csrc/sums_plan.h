// sums_plan.h — the chunk plan of a proof over checksummed POST data (b200post_generate_proof_sums, DESIGN.md §5): the
// POST's labels cut into digest ranges, whole ranges packed into chunks and whole chunks into shards, so that no digest
// range ever straddles a chunk, a shard or a device.  Plain C++17, so that it can be tested on the CPU; prover.cu streams
// the chunks.
#pragma once
#include <cstddef>
#include <cstdint>
#include <utility>
#include <vector>

namespace b200post {

// One postdata file as the plan sees it: its labels, and the prefix [0, covered) its usable sidecar describes with one
// 32-byte digest per range (covered = 0 and digests = nullptr without one).
struct SumsFile { uint64_t labels, covered; const uint8_t *digests; };

// Global labels [first, first + count) of one file: a sidecar's digest range (sum = its 32 bytes), or a piece of the file
// no digest covers (sum = nullptr), cut on the same 2^16-label grid.
struct SumRange { uint64_t first, count; const uint8_t *sum; };

// Global labels [first, first + count), made of the plan's ranges [r0, r1)
struct SumChunk { uint64_t first, count; size_t r0, r1; };

struct SumsPlan {
    std::vector<SumRange> ranges;                    // ascending, tiling [0, numLabels)
    std::vector<SumChunk> chunks;                    // ascending, tiling [0, numLabels)
    std::vector<std::pair<size_t, size_t>> shards;   // per shard: its chunks [first, end) (a shard may have none)
    uint64_t max_chunk = 0;                          // labels of the largest chunk
    size_t max_ranges = 0;                           // ranges of the chunk with the most
    // shard s's labels [lo, hi) (lo == hi for a shard without chunks)
    std::pair<uint64_t, uint64_t> shard_labels(size_t s) const;
};

// The files in order (file f's first label is the sum of the earlier files' labels).  Range boundaries are file starts,
// every 2^16 labels within a file and each covered end.  A chunk is a run of whole ranges of at most
// max(chunk_labels, 2^16) labels, packed greedily from label 0; the chunks are split into n_shards contiguous shards
// whose chunk counts differ by at most one, the earlier shards taking the odd chunks.
SumsPlan plan_sums(const std::vector<SumsFile> &files, uint64_t chunk_labels, size_t n_shards);

}  // namespace b200post
