// prove_rule.h — the proving scan's rule without the devices (DESIGN.md §5): the shards' hit books, the stop rule, the
// saturation plan, the window decision and applying a recheck result.  Plain C++17, so that it can be driven on the CPU;
// ShardedScan (prover.cu) runs it with host threads, Scanners and the device recheck, the initial proof
// (initial_proof.cu) decides with it.
#pragma once
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <set>
#include <utility>
#include <vector>

namespace b200post {

// A kept hit: its stored bytes (checked scan only), and whether they are known to equal the recomputed label (good) or
// not yet looked at (pending).  A damaged hit is removed from its list.
struct KeptHit { uint64_t index; uint8_t label[16]; bool good; };

// One shard's hits per absolute nonce of the pass, ascending index, and its labels scanned (the prefix whose hits are in
// the book).  Unchecked, hits are born good and a nonce keeps its first K2; checked, they are born pending and all are
// kept, since dropping a damaged hit can make the next one count.
class HitBook {
public:
    using Lists = std::map<uint32_t, std::vector<KeptHit>>;   // ordered, so ties resolve to the lower nonce

    HitBook(uint32_t nonces, uint32_t k2, bool born_good) : nonces_(nonces), k2_(k2), born_good_(born_good) {}
    // a hit above every earlier hit of its nonce; `label`: its 16 stored bytes, or nullptr.  good: known to be the
    // real label already (a checksummed proof's covered hit), even in a book whose hits are born pending
    void add(uint32_t nonce, uint64_t index, const uint8_t *label, bool good = false);
    void advance(uint64_t labels) { scanned_ += labels; }
    // a recheck's verdict on a hit, if it is still kept: good, or damaged and removed
    void settle(uint32_t nonce, uint64_t index, bool damaged);
    bool full() const { return full_ == nonces_; }   // every nonce has K2 kept hits
    // every nonce has K2 good hits: later labels change no nonce's first K2 usable hits
    bool saturated() const;
    const Lists &lists() const { return lists_; }
    uint64_t scanned() const { return scanned_; }

private:
    Lists lists_;
    uint32_t nonces_, k2_, full_ = 0;   // full_: nonces with K2 kept hits
    bool born_good_;
    uint64_t scanned_ = 0;
};

// A pending hit for a recheck round: its shard, nonce, index and stored bytes.
struct RecheckItem {
    RecheckItem(size_t s, uint32_t n, const KeptHit &k) : shard(s), nonce(n), index(k.index) { std::memcpy(label, k.label, 16); }
    size_t shard; uint32_t nonce; uint64_t index; uint8_t label[16];
};

// One pass of a proof: the nonce windows [first + w·window, first + (w+1)·window), w < windows, over contiguous label
// shards in order, one hit book each.  x is the end of the longest gap-free scanned prefix of the labels, a saturated
// shard counting as whole.  The scan stops once the selection rule's winner over the hits below x of the pass's lowest
// window has its first K2 hits all good; recheck rounds settle its pending ones first.  A shard also stops once it is
// saturated, after a round over its pending hits among each nonce's first K2 once every nonce has K2 kept.  Unchecked,
// every hit is born good and no round ever runs.
class ProveRule {
public:
    // The recheck: the labels of `items` recomputed on shard `shard`'s device and compared with their stored bytes;
    // bad[i] = 1 where item i differs.  Returns a status (B200POST_OK = 0).
    using Recheck = std::function<int(size_t shard, const std::vector<RecheckItem> &items, std::vector<uint8_t> *bad)>;

    // ranges[s]: shard s's labels [lo, hi).  With a recheck (the checked proof) hits are born pending, without it good.
    ProveRule(const std::vector<std::pair<uint64_t, uint64_t>> &ranges, uint32_t first, uint32_t window, uint32_t windows,
              uint32_t k2, Recheck recheck = nullptr);

    HitBook &book(size_t s) { return shards_[s].book; }
    // Shard s's thread after each chunk, under `mu` (which guards every book while threads run): whether the shard
    // stops.  `mu` is released while a recheck runs.  One winner round runs at a time; a saturation round touches only
    // its own shard's hits.  *rc: a failed recheck's status.
    bool should_stop(size_t s, std::mutex &mu, int *rc);
    // After the scan, per window of the pass in order: recheck rounds (on shard 0's device) until the window's winner has
    // its first K2 hits all good (true: the winner and its indices) or no nonce of it has K2 usable hits (the next
    // window).  False with *rc OK when no window has one.  Needs no round when the scan stopped on a decision.
    bool decide(uint32_t *nonce, std::vector<uint64_t> *indices, int *rc);

    uint64_t scanned() const;   // over every shard
    uint64_t rechecked() const { return rechecked_; }
    uint32_t rounds() const { return rounds_; }
    const std::set<uint64_t> &damaged() const { return damaged_; }

private:
    struct Shard { HitBook book; uint64_t size; };
    enum Plan { NONE, DECIDED, RECHECK };

    Plan plan_winner(uint32_t w, std::vector<RecheckItem> *items, uint32_t *nonce, std::vector<uint64_t> *indices) const;
    bool plan_saturation(size_t s, std::vector<RecheckItem> *items) const;
    int round(size_t s, const std::vector<RecheckItem> &items, std::unique_lock<std::mutex> *lk);

    std::vector<Shard> shards_;
    uint32_t first_, window_, windows_, k2_;
    Recheck recheck_;
    bool decided_ = false, round_busy_ = false;
    uint64_t rechecked_ = 0;
    uint32_t rounds_ = 0;
    std::set<uint64_t> damaged_;
};

}  // namespace b200post
