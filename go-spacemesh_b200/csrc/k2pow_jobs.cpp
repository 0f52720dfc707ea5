// k2pow_jobs.cpp — see k2pow_jobs.h.
#include "k2pow_jobs.h"

#include <algorithm>

namespace b200post {

namespace {
constexpr uint64_t kNonceSpace = 1ull << 56;   // the input carries 7 bytes of pow
}

JobSchedule::JobSchedule(size_t n_jobs, uint64_t cap)
    : cap_(cap == 0 || cap > kNonceSpace ? kNonceSpace : cap), best_(n_jobs, kNotFound), final_(n_jobs, false) {}

bool JobSchedule::take(uint64_t batch, Window *w) {
    w->jobs.clear();
    for (uint32_t j = 0; j < best_.size(); j++) if (best_[j] == kNotFound) w->jobs.push_back(j);
    if (w->jobs.empty() || next_ >= cap_) return false;
    w->per = std::min<uint64_t>(std::max<uint64_t>(1, batch / w->jobs.size()), cap_ - next_);
    w->lo = next_;
    w->id = ids_++;
    next_ += w->per;
    hashes_ += w->jobs.size() * w->per;
    inflight_[w->id] = *w;
    return true;
}

std::vector<std::vector<JobSegment>> JobSchedule::batches(const Window &w, uint64_t batch) {
    std::vector<std::vector<JobSegment>> out;
    const uint64_t total = w.jobs.size() * w.per;
    for (uint64_t b0 = 0; b0 < total; b0 += batch) {
        const uint64_t b1 = std::min(total, b0 + batch);
        std::vector<JobSegment> segs;
        for (uint64_t v = b0; v < b1;) {
            const uint64_t i = v / w.per, in_job = v - i * w.per, cnt = std::min(w.per - in_job, b1 - v);
            segs.push_back(JobSegment{(uint32_t)(v - b0), (uint32_t)cnt, w.jobs[i], 0, w.lo + in_job});
            v += cnt;
        }
        out.push_back(std::move(segs));
    }
    return out;
}

bool JobSchedule::is_final(uint32_t j) const {
    // a window still running that holds j and starts at or below j's lowest hit may still lower it
    for (const auto &kv : inflight_)
        if (kv.second.lo <= best_[j] && std::binary_search(kv.second.jobs.begin(), kv.second.jobs.end(), j)) return false;
    return best_[j] != kNotFound || next_ >= cap_;
}

std::vector<uint32_t> JobSchedule::newly_final(const std::vector<uint32_t> &candidates) {
    std::vector<uint32_t> out;
    for (uint32_t j : candidates)
        if (!final_[j] && is_final(j)) { final_[j] = true; out.push_back(j); }
    return out;
}

std::vector<uint32_t> JobSchedule::finish(const Window &w, const std::vector<uint64_t> &hits) {
    inflight_.erase(w.id);
    for (size_t i = 0; i < w.jobs.size(); i++) best_[w.jobs[i]] = std::min(best_[w.jobs[i]], hits[i]);
    return newly_final(w.jobs);
}

std::vector<uint32_t> JobSchedule::settle() {
    std::vector<uint32_t> all(best_.size());
    for (uint32_t j = 0; j < all.size(); j++) all[j] = j;
    return newly_final(all);
}

}  // namespace b200post
