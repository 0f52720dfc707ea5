// sums_plan_emul.cpp — csrc/sums_plan.cpp's chunk plan behind a flat C interface, for tests/test_prove_sums_host.py.
#include <cstdint>
#include <vector>

#include "../go-spacemesh_b200/csrc/sums_plan.h"

using namespace b200post;

// Files f < n_files of labels[f] labels, covered[f] of them by a sidecar whose digests are slots digest_first[f] + k of
// one table.  Outputs (each row 4 x u64), at most `cap` rows each:
//   ranges: first, count, covered (0/1), digest slot (~0 when uncovered)
//   chunks: first, count, r0, r1
//   shards (n_shards rows): first chunk, end chunk, lo, hi
//   counts: ranges, chunks, max_chunk, max_ranges
// Returns 0, or -1 when a table would exceed cap.
extern "C" int emul_plan(uint32_t n_files, const uint64_t *labels, const uint64_t *covered, const uint64_t *digest_first,
                         uint64_t chunk_labels, uint32_t n_shards, uint64_t cap, uint64_t *ranges, uint64_t *chunks,
                         uint64_t *shards, uint64_t *counts) {
    uint64_t slots = 0;
    for (uint32_t f = 0; f < n_files; f++) {
        const uint64_t end = digest_first[f] + (covered[f] + 65535) / 65536;
        if (end > slots) slots = end;
    }
    std::vector<uint8_t> table((size_t)(slots + 1) * 32);
    std::vector<SumsFile> files;
    for (uint32_t f = 0; f < n_files; f++)
        files.push_back({labels[f], covered[f], covered[f] ? table.data() + digest_first[f] * 32 : nullptr});
    const SumsPlan p = plan_sums(files, chunk_labels, n_shards);
    if (p.ranges.size() > cap || p.chunks.size() > cap) return -1;
    for (size_t i = 0; i < p.ranges.size(); i++) {
        const SumRange &r = p.ranges[i];
        uint64_t *o = ranges + 4 * i;
        o[0] = r.first; o[1] = r.count; o[2] = r.sum != nullptr;
        o[3] = r.sum ? (uint64_t)(r.sum - table.data()) / 32 : ~0ull;
    }
    for (size_t i = 0; i < p.chunks.size(); i++) {
        const SumChunk &c = p.chunks[i];
        uint64_t *o = chunks + 4 * i;
        o[0] = c.first; o[1] = c.count; o[2] = c.r0; o[3] = c.r1;
    }
    for (size_t s = 0; s < p.shards.size(); s++) {
        const auto lh = p.shard_labels(s);
        uint64_t *o = shards + 4 * s;
        o[0] = p.shards[s].first; o[1] = p.shards[s].second; o[2] = lh.first; o[3] = lh.second;
    }
    counts[0] = p.ranges.size(); counts[1] = p.chunks.size(); counts[2] = p.max_chunk; counts[3] = p.max_ranges;
    return 0;
}
