// sums_plan.cpp — see sums_plan.h.
#include "sums_plan.h"

#include <algorithm>

namespace b200post {

namespace {
constexpr uint64_t kRangeLabels = 1ull << 16;   // kSumBlockLabels (postdata_io.h)
}

std::pair<uint64_t, uint64_t> SumsPlan::shard_labels(size_t s) const {
    const auto &sh = shards[s];
    if (sh.first == sh.second) {
        const uint64_t at = sh.first < chunks.size() ? chunks[sh.first].first : chunks.empty() ? 0 : chunks.back().first + chunks.back().count;
        return {at, at};
    }
    return {chunks[sh.first].first, chunks[sh.second - 1].first + chunks[sh.second - 1].count};
}

SumsPlan plan_sums(const std::vector<SumsFile> &files, uint64_t chunk_labels, size_t n_shards) {
    SumsPlan p;
    uint64_t base = 0;
    for (const SumsFile &f : files) {
        const uint64_t covered = std::min(f.covered, f.labels);
        for (uint64_t pos = 0; pos < f.labels;) {
            const uint64_t grid = pos / kRangeLabels * kRangeLabels + kRangeLabels;
            const bool in = pos < covered;
            const uint64_t end = std::min(grid, in ? covered : f.labels);
            p.ranges.push_back({base + pos, end - pos, in ? f.digests + pos / kRangeLabels * 32 : nullptr});
            pos = end;
        }
        base += f.labels;
    }
    const uint64_t bound = std::max(chunk_labels, kRangeLabels);
    for (size_t r = 0; r < p.ranges.size(); r++) {
        const SumRange &x = p.ranges[r];
        if (p.chunks.empty() || p.chunks.back().count + x.count > bound) p.chunks.push_back({x.first, 0, r, r});
        SumChunk &c = p.chunks.back();
        c.count += x.count;
        c.r1 = r + 1;
    }
    for (const SumChunk &c : p.chunks) {
        p.max_chunk = std::max(p.max_chunk, c.count);
        p.max_ranges = std::max(p.max_ranges, c.r1 - c.r0);
    }
    const size_t n = std::max<size_t>(n_shards, 1), q = p.chunks.size() / n, rem = p.chunks.size() % n;
    for (size_t s = 0; s < n; s++) {
        const size_t first = s * q + std::min(s, rem);
        p.shards.push_back({first, first + q + (s < rem ? 1 : 0)});
    }
    return p;
}

}  // namespace b200post
