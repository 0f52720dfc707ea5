// prove_rule_emul.cpp — drives the prover's rule (csrc/prove_rule.cpp) on the CPU: one pass over given hits, chunk by
// chunk in a chosen shard order, with the stop rule after every chunk, the decision at the end, and a recheck that reads
// a damage mask instead of recomputing labels.  Test infrastructure; tests/test_prove_rule_host.py builds it with g++.
#include <algorithm>
#include <mutex>
#include <vector>

#include "../go-spacemesh_b200/csrc/prove_rule.h"

using namespace b200post;

// Shard s holds the labels [bounds[s], bounds[s + 1]).  order 0: one chunk of every live shard per round, ascending shard
// order; 1: the same, descending; 2: shard by shard from the last, each until it ends or stops.  hits: (nonce, index) of
// the pass's nonces, ascending (index, nonce).  damaged: one byte per label, 1 = damaged, or nullptr for the unchecked
// rule.  Returns 1 with (*nonce, indices[0 .. k2)) when the pass has a proof, 0 when not, -status on a recheck failure;
// stats = {labels scanned, labels rechecked, rounds, hits the recheck reported damaged}.
extern "C" int emul_pass(uint32_t n_shards, const uint64_t *bounds, uint64_t chunk, int order, uint32_t first, uint32_t window,
                         uint32_t windows, uint32_t k2, const uint32_t *hit_nonce, const uint64_t *hit_index, uint64_t n_hits,
                         const uint8_t *damaged, uint32_t *nonce, uint64_t *indices, uint64_t *stats) {
    std::vector<std::pair<uint64_t, uint64_t>> ranges;
    for (uint32_t s = 0; s < n_shards; s++) ranges.push_back({bounds[s], bounds[s + 1]});
    uint64_t bad_hits = 0;
    ProveRule::Recheck recheck = nullptr;
    if (damaged)
        recheck = [&](size_t, const std::vector<RecheckItem> &items, std::vector<uint8_t> *bad) {
            for (size_t i = 0; i < items.size(); i++) bad_hits += (*bad)[i] = damaged[items[i].index];
            return 0;
        };
    ProveRule rule(ranges, first, window, windows, k2, recheck);
    std::mutex mu;
    std::vector<uint64_t> pos(bounds, bounds + n_shards);
    std::vector<bool> stopped(n_shards, false);
    // one chunk of shard s folded and the stop rule run: 1, or 0 when the shard had ended or stopped, or -status
    auto step = [&](uint32_t s) {
        if (stopped[s] || pos[s] == bounds[s + 1]) return 0;
        const uint64_t end = std::min(bounds[s + 1], pos[s] + chunk);
        const uint64_t *lo = std::lower_bound(hit_index, hit_index + n_hits, pos[s]);
        const uint64_t *hi = std::lower_bound(hit_index, hit_index + n_hits, end);
        for (const uint64_t *h = lo; h < hi; h++) rule.book(s).add(hit_nonce[h - hit_index], *h, nullptr);
        rule.book(s).advance(end - pos[s]);
        pos[s] = end;
        int rc = 0;
        stopped[s] = rule.should_stop(s, mu, &rc);
        return rc ? -rc : 1;
    };
    int rc = 0;
    if (order == 2) {
        for (uint32_t s = n_shards; rc >= 0 && s-- > 0;)
            while ((rc = step(s)) > 0) {}
    } else {
        for (bool any = true; any;) {
            any = false;
            for (uint32_t i = 0; i < n_shards && rc >= 0; i++) any |= (rc = step(order ? n_shards - 1 - i : i)) > 0;
        }
    }
    if (rc < 0) return rc;
    std::vector<uint64_t> idx;
    const bool have = rule.decide(nonce, &idx, &rc);
    if (rc) return -rc;
    std::copy(idx.begin(), idx.end(), indices);
    stats[0] = rule.scanned(); stats[1] = rule.rechecked(); stats[2] = rule.rounds(); stats[3] = bad_hits;
    return have;
}
