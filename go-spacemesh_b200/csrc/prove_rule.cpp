// prove_rule.cpp — see prove_rule.h.
#include "prove_rule.h"

#include <algorithm>
#include <cstring>

#include "../../include/b200post.h"

namespace b200post {

void HitBook::add(uint32_t nonce, uint64_t index, const uint8_t *label, bool good) {
    std::vector<KeptHit> &l = lists_[nonce];
    if (born_good_ && l.size() >= k2_) return;   // hits past a nonce's K2-th good one never count
    KeptHit k{index, {}, born_good_ || good};
    if (label) memcpy(k.label, label, 16);
    l.push_back(k);
    full_ += l.size() == k2_;
}

void HitBook::settle(uint32_t nonce, uint64_t index, bool damaged) {
    std::vector<KeptHit> &l = lists_[nonce];
    const auto it = std::lower_bound(l.begin(), l.end(), index, [](const KeptHit &k, uint64_t v) { return k.index < v; });
    if (it == l.end() || it->index != index) return;
    if (!damaged) { it->good = true; return; }
    full_ -= l.size() == k2_;
    l.erase(it);
}

bool HitBook::saturated() const {
    if (!full()) return false;
    if (born_good_) return true;
    for (const auto &kv : lists_) {
        uint32_t good = 0;
        for (const KeptHit &k : kv.second) if ((good += k.good) == k2_) break;
        if (good < k2_) return false;
    }
    return true;
}

ProveRule::ProveRule(const std::vector<std::pair<uint64_t, uint64_t>> &ranges, uint32_t first, uint32_t window, uint32_t windows,
                     uint32_t k2, Recheck recheck)
    : first_(first), window_(window), windows_(windows), k2_(k2), recheck_(std::move(recheck)) {
    for (const auto &r : ranges) shards_.push_back({HitBook(window * windows, k2, !recheck_), r.second - r.first});
}

uint64_t ProveRule::scanned() const {
    uint64_t t = 0;
    for (const Shard &sh : shards_) t += sh.book.scanned();
    return t;
}

// Under the lock (or with the threads joined).  The selection rule over the kept (good and pending) hits below x of the
// nonces of window w of the pass, each nonce's first K2 of them in shard order: among nonces with K2, the lowest K2-th
// index wins; ties go to the lower nonce.  NONE if no nonce has K2; DECIDED with the winner when its first K2 are all
// good; RECHECK with its pending ones.
ProveRule::Plan ProveRule::plan_winner(uint32_t w, std::vector<RecheckItem> *items, uint32_t *nonce,
                                       std::vector<uint64_t> *indices) const {
    size_t below = 0;   // the shards that hold hits below x
    while (below < shards_.size()) {
        const Shard &sh = shards_[below++];
        if (sh.book.scanned() < sh.size && !sh.book.saturated()) break;   // x lies in this shard
    }
    struct Ref { size_t shard; const KeptHit *k; };
    std::vector<Ref> best, cur;
    uint32_t win = 0;
    for (uint32_t n = first_ + w * window_; n < first_ + (w + 1) * window_; n++) {
        cur.clear();
        for (size_t s = 0; s < below && cur.size() < k2_; s++) {
            const HitBook::Lists &l = shards_[s].book.lists();
            const auto kv = l.find(n);
            if (kv == l.end()) continue;
            for (size_t i = 0; i < kv->second.size() && cur.size() < k2_; i++) cur.push_back({s, &kv->second[i]});
        }
        if (cur.size() == k2_ && (best.empty() || cur.back().k->index < best.back().k->index)) { best.swap(cur); win = n; }
    }
    if (best.empty()) return NONE;
    for (const Ref &r : best) if (!r.k->good) items->emplace_back(r.shard, win, *r.k);
    if (!items->empty()) return RECHECK;
    *nonce = win;
    indices->clear();
    for (const Ref &r : best) indices->push_back(r.k->index);
    return DECIDED;
}

// Under the lock: when every nonce has K2 kept hits in shard s but not K2 good ones, the pending ones among each nonce's
// first K2 in the shard (a shard's own saturation stop counts good hits only).
bool ProveRule::plan_saturation(size_t s, std::vector<RecheckItem> *items) const {
    const HitBook &b = shards_[s].book;
    if (!b.full()) return false;
    for (const auto &kv : b.lists())
        for (size_t i = 0; i < kv.second.size() && i < k2_; i++)
            if (!kv.second[i].good) items->emplace_back(s, kv.first, kv.second[i]);
    return !items->empty();
}

// One recheck round: the recheck with `lk` released (when given), then, under it, good hits marked and damaged ones
// dropped.
int ProveRule::round(size_t s, const std::vector<RecheckItem> &items, std::unique_lock<std::mutex> *lk) {
    std::vector<uint8_t> bad(items.size(), 0);
    if (lk) lk->unlock();
    const int rc = recheck_(s, items, &bad);
    if (lk) lk->lock();
    if (rc) return rc;
    for (size_t i = 0; i < items.size(); i++) {
        shards_[items[i].shard].book.settle(items[i].nonce, items[i].index, bad[i]);
        if (bad[i]) damaged_.insert(items[i].index);
    }
    rechecked_ += items.size(); rounds_++;
    return B200POST_OK;
}

bool ProveRule::should_stop(size_t s, std::mutex &mu, int *rc) {
    std::unique_lock<std::mutex> lk(mu);
    for (;;) {
        if (decided_ || shards_[s].book.saturated()) return true;
        std::vector<RecheckItem> items;
        bool winner_round = false;
        if (!round_busy_) {
            uint32_t nonce;
            std::vector<uint64_t> idx;
            const Plan p = plan_winner(0, &items, &nonce, &idx);   // the pass's lowest window decides the stop
            if (p == DECIDED) { decided_ = true; return true; }
            winner_round = round_busy_ = p == RECHECK;
        }
        if (!winner_round && !plan_saturation(s, &items)) return false;
        *rc = round(s, items, &lk);
        if (winner_round) round_busy_ = false;
        if (*rc) return true;
    }
}

bool ProveRule::decide(uint32_t *nonce, std::vector<uint64_t> *indices, int *rc) {
    *rc = B200POST_OK;
    for (uint32_t w = 0; w < windows_; w++)
        for (;;) {
            std::vector<RecheckItem> items;
            const Plan p = plan_winner(w, &items, nonce, indices);
            if (p == DECIDED) return true;
            if (p == NONE) break;
            if ((*rc = round(0, items, nullptr))) return false;
        }
    return false;
}

}  // namespace b200post
