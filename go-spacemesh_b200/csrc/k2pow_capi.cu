// k2pow_capi.cu — extern "C" surface of the k2pow (RandomX) engine (declared in include/b200post_k2pow.h).
#include <algorithm>
#include <atomic>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b200post_k2pow.h"
#include "engine.h"
#include "k2pow_jobs.h"
#include "proof_common.h"
#include "randomx_engine.h"

using namespace b200post;

namespace {

std::string key_of(const uint8_t *key, size_t len) {
    if (!key) return std::string(B200POST_K2POW_DEFAULT_KEY);
    return std::string(reinterpret_cast<const char *>(key), len);
}

rx::K2powTemplate template_of(const b200post_k2pow_params *p) {
    rx::K2powTemplate t{};
    t.tail[0] = p->nonce_group;
    memcpy(t.tail + 1, p->challenge8, 8);
    memcpy(t.tail + 9, p->node_id, 32);
    t.start = 0;
    return t;
}

constexpr uint64_t kNonceSpace = 1ull << 56;   // the input carries 7 bytes of pow

bool clamp_range(uint64_t start, uint64_t &count) {
    if (start >= kNonceSpace) return false;
    if (count > kNonceSpace - start) count = kNonceSpace - start;
    return true;
}

// The jobs of groups first_group .. first_group + n_groups - 1 of one identity (p->nonce_group is not used)
std::vector<K2powJob> group_jobs(const b200post_k2pow_params *p, uint32_t first_group, uint32_t n_groups) {
    std::vector<K2powJob> jobs(n_groups);
    for (uint32_t g = 0; g < n_groups; g++) {
        rx::K2powTemplate t = template_of(p);
        t.tail[0] = (uint8_t)(first_group + g);   // the absolute group number is the k2pow input's group byte
        memcpy(jobs[g].tail, t.tail, 41);
        memcpy(jobs[g].difficulty, p->difficulty, 32);
    }
    return jobs;
}

}  // namespace

namespace b200post {

int k2pow_search_jobs(const std::vector<RandomxEngine *> &eng, const std::string &key, const std::vector<K2powJob> &jobs, uint64_t cap,
                      uint64_t *pows, uint64_t *hashes_done, const volatile int *cancel, const std::function<void(uint32_t, uint64_t)> &on_final) {
    JobSchedule sched(jobs.size(), cap);
    std::mutex mu;                     // guards sched and orders the on_final calls
    std::atomic<bool> stop{false};
    for (RandomxEngine *e : eng) e->reset_timing();
    const auto report = [&](const std::vector<uint32_t> &done) { if (on_final) for (uint32_t j : done) on_final(j, sched.pow(j)); };
    const auto part = [&](size_t i) -> int {
        uint64_t batch = 0;
        eng[i]->batch_size(&batch);
        JobSchedule::Window w;
        std::vector<uint64_t> hits;
        std::vector<uint32_t> slot;
        while (!stop) {
            if (cancel && *cancel) { set_error("cancelled"); return B200POST_ERR_CANCELLED; }
            {
                std::lock_guard<std::mutex> lk(mu);
                if (!sched.take(batch, &w)) { report(sched.settle()); break; }
            }
            hits.assign(w.jobs.size(), B200POST_K2POW_NOT_FOUND);
            for (const std::vector<JobSegment> &segs : JobSchedule::batches(w, batch)) {
                slot.resize(segs.size());
                if (int rc = eng[i]->search_segments(key, jobs.data(), jobs.size(), segs.data(), segs.size(), slot.data())) return rc;
                for (size_t s = 0; s < segs.size(); s++) {
                    if (slot[s] == 0xffffffffu) continue;
                    const size_t k = (size_t)(std::lower_bound(w.jobs.begin(), w.jobs.end(), segs[s].job) - w.jobs.begin());
                    hits[k] = std::min(hits[k], segs[s].first_pow + slot[s]);
                }
            }
            std::lock_guard<std::mutex> lk(mu);
            report(sched.finish(w, hits));
        }
        return B200POST_OK;
    };
    const int rc = eng.size() == 1 ? part(0) : fan_out(eng.size(), [&](size_t i) {
        const int r = part(i);
        if (r != B200POST_OK) stop = true;
        return r;
    });
    for (size_t j = 0; j < jobs.size(); j++) pows[j] = sched.final(j) ? sched.pow(j) : B200POST_K2POW_NOT_FOUND;
    if (hashes_done) *hashes_done = sched.hashes();
    return rc;
}

}  // namespace b200post

extern "C" {

void b200post_k2pow_scale_difficulty(const uint8_t pow_difficulty[32], uint32_t num_units, uint8_t out[32]) {
    // the prover and the verifier scale with the same division
    div256_u32(pow_difficulty, num_units ? num_units : 1, out);
}

int b200post_randomx_prepare(uint32_t provider, const uint8_t *key, size_t key_len) {
    RandomxEngine *e;
    if (int rc = randomx_engine(provider, &e)) return rc;
    return e->prepare(key_of(key, key_len));
}

int b200post_randomx_hash(uint32_t provider, const uint8_t *key, size_t key_len, const uint8_t *inputs, size_t input_len, size_t n,
                          uint8_t *out32) {
    if ((n && !out32) || (n && input_len && !inputs) || input_len > (1u << 20)) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    RandomxEngine *e;
    if (int rc = randomx_engine(provider, &e)) return rc;
    return e->hash_inputs(key_of(key, key_len), inputs, input_len, n, out32);
}

int b200post_randomx_dataset_read(uint32_t provider, const uint8_t *key, size_t key_len, uint64_t first_item, uint64_t count,
                                  uint64_t *out) {
    if ((count && !out) || first_item > rx::kDatasetItems || count > rx::kDatasetItems - first_item) {
        set_error("invalid argument: items past the end of the dataset, or no output buffer");
        return B200POST_ERR_INVALID_ARGUMENT;
    }
    RandomxEngine *e;
    if (int rc = randomx_engine(provider, &e)) return rc;
    return e->dataset_read(key_of(key, key_len), first_item, count, out);
}

int b200post_k2pow_hashes(uint32_t provider, const b200post_k2pow_params *p, uint64_t start, uint64_t count, uint8_t *out32) {
    if (!p || (count && !out32) || !clamp_range(start, count)) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    RandomxEngine *e;
    if (int rc = randomx_engine(provider, &e)) return rc;
    return e->k2pow(key_of(p->cache_key, p->cache_key_len), template_of(p), nullptr, start, count, out32, nullptr, nullptr, nullptr);
}

int b200post_k2pow_search(uint32_t provider, const b200post_k2pow_params *p, uint64_t start, uint64_t count, uint64_t *found,
                          uint64_t *hashes_done, const volatile int *cancel) {
    if (!p || !found || !clamp_range(start, count)) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    RandomxEngine *e;
    if (int rc = randomx_engine(provider, &e)) return rc;
    return e->k2pow(key_of(p->cache_key, p->cache_key_len), template_of(p), p->difficulty, start, count, nullptr, found, hashes_done, cancel);
}

int b200post_k2pow_search_multi(const uint32_t *providers, int n_providers, const b200post_k2pow_params *p, uint64_t start,
                                uint64_t count, uint64_t *found, uint64_t *hashes_done, const volatile int *cancel) {
    if (!providers || n_providers <= 0 || !p || !found || !clamp_range(start, count)) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    if (n_providers == 1) return b200post_k2pow_search(providers[0], p, start, count, found, hashes_done, cancel);
    std::vector<RandomxEngine *> eng;
    if (int rc = randomx_engines(providers, n_providers, &eng)) return rc;
    uint64_t batch = UINT64_MAX;
    for (RandomxEngine *e : eng) {
        uint64_t b = 0;
        e->batch_size(&b);
        batch = std::min(batch, b);
    }
    // device i takes batches i, i+n, i+2n, ... of `batch` nonces; everyone stops after the round in which a hit appears
    const std::string key = key_of(p->cache_key, p->cache_key_len);
    const rx::K2powTemplate tmpl = template_of(p);
    std::vector<uint64_t> hits(n_providers, UINT64_MAX), dones(n_providers, 0);
    volatile int any_hit = 0;
    const int rc = fan_out((size_t)n_providers, [&](size_t i) -> int {
        if ((uint64_t)i * batch >= count) return B200POST_OK;
        const int r = eng[i]->k2pow(key, tmpl, p->difficulty, start + (uint64_t)i * batch, count - (uint64_t)i * batch, nullptr, &hits[i],
                                    &dones[i], cancel, batch * (uint64_t)n_providers, &any_hit);
        if (hits[i] != UINT64_MAX) any_hit = 1;
        return r;
    });
    *found = UINT64_MAX;
    uint64_t total = 0;
    for (int i = 0; i < n_providers; i++) { total += dones[i]; if (hits[i] < *found) *found = hits[i]; }
    if (hashes_done) *hashes_done = total;
    return rc;
}

int b200post_k2pow_search_groups(uint32_t provider, const b200post_k2pow_params *p, uint32_t n_groups, uint64_t max_nonces_per_group,
                                 uint64_t *pows, uint64_t *hashes_done, const volatile int *cancel) {
    return b200post_k2pow_search_group_range(provider, p, 0, n_groups, max_nonces_per_group, pows, hashes_done, cancel);
}

int b200post_k2pow_search_group_range(uint32_t provider, const b200post_k2pow_params *p, uint32_t first_group, uint32_t n_groups,
                                      uint64_t max_nonces_per_group, uint64_t *pows, uint64_t *hashes_done, const volatile int *cancel) {
    if (!p || !pows || n_groups == 0 || (uint64_t)first_group + n_groups > 256) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    RandomxEngine *e;
    if (int rc = randomx_engine(provider, &e)) return rc;
    return k2pow_search_jobs({e}, key_of(p->cache_key, p->cache_key_len), group_jobs(p, first_group, n_groups), max_nonces_per_group, pows,
                             hashes_done, cancel);
}

int b200post_k2pow_search_groups_multi(const uint32_t *providers, int n_providers, const b200post_k2pow_params *p,
                                       uint32_t n_groups, uint64_t max_nonces_per_group, uint64_t *pows,
                                       uint64_t *hashes_done, const volatile int *cancel) {
    return b200post_k2pow_search_group_range_multi(providers, n_providers, p, 0, n_groups, max_nonces_per_group, pows, hashes_done, cancel);
}

int b200post_k2pow_search_group_range_multi(const uint32_t *providers, int n_providers, const b200post_k2pow_params *p,
                                            uint32_t first_group, uint32_t n_groups, uint64_t max_nonces_per_group, uint64_t *pows,
                                            uint64_t *hashes_done, const volatile int *cancel) {
    if (!providers || n_providers <= 0 || !p || !pows || n_groups == 0 || (uint64_t)first_group + n_groups > 256) {
        set_error("invalid argument");
        return B200POST_ERR_INVALID_ARGUMENT;
    }
    if (n_providers == 1) return b200post_k2pow_search_group_range(providers[0], p, first_group, n_groups, max_nonces_per_group, pows, hashes_done, cancel);
    std::vector<RandomxEngine *> eng;
    if (int rc = randomx_engines(providers, n_providers, &eng)) return rc;
    return k2pow_search_jobs(eng, key_of(p->cache_key, p->cache_key_len), group_jobs(p, first_group, n_groups), max_nonces_per_group, pows,
                             hashes_done, cancel);
}

int b200post_k2pow_search_jobs(const uint32_t *providers, int n_providers, const uint8_t *cache_key, size_t cache_key_len,
                               size_t n_jobs, const b200post_k2pow_job *jobs, uint64_t max_nonces_per_job, uint64_t *pows,
                               uint64_t *hashes_done, const volatile int *cancel) {
    if (!providers || n_providers <= 0 || n_jobs == 0 || !jobs || !pows) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    std::vector<RandomxEngine *> eng;
    if (int rc = randomx_engines(providers, n_providers, &eng)) return rc;
    std::vector<K2powJob> table(n_jobs);
    for (size_t j = 0; j < n_jobs; j++) {
        table[j].tail[0] = jobs[j].nonce_group;
        memcpy(table[j].tail + 1, jobs[j].challenge8, 8);
        memcpy(table[j].tail + 9, jobs[j].node_id, 32);
        memcpy(table[j].difficulty, jobs[j].difficulty, 32);
    }
    return k2pow_search_jobs(eng, key_of(cache_key, cache_key_len), table, max_nonces_per_job, pows, hashes_done, cancel);
}

int b200post_k2pow_verify(uint32_t provider, const b200post_k2pow_params *p, uint64_t pow, int *valid) {
    if (!p || !valid) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    *valid = 0;
    if (pow >= kNonceSpace) return B200POST_OK;     // does not fit the 7 input bytes: cannot be what the prover hashed
    RandomxEngine *e;
    if (int rc = randomx_engine(provider, &e)) return rc;
    uint64_t found = UINT64_MAX;
    const int rc = e->k2pow(key_of(p->cache_key, p->cache_key_len), template_of(p), p->difficulty, pow, 1, nullptr, &found, nullptr, nullptr);
    if (rc == B200POST_OK) *valid = found == pow;
    return rc;
}

int b200post_randomx_last_timing(uint32_t provider, double *total_ms, double *vm_kernel_ms, uint64_t *hashes, uint64_t *vm_launches) {
    RandomxEngine *e = randomx_engine_for(provider);
    if (!e) return B200POST_ERR_NO_DEVICE;
    e->last_timing(total_ms, vm_kernel_ms, hashes, vm_launches);
    return B200POST_OK;
}

int b200post_randomx_batch_size(uint32_t provider, uint64_t *vms) {
    RandomxEngine *e = randomx_engine_for(provider);
    if (!e) return B200POST_ERR_NO_DEVICE;
    return e->batch_size(vms);
}

}  // extern "C"
