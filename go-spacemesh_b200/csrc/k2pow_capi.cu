// k2pow_capi.cu — extern "C" surface of the k2pow (RandomX) engine (declared in include/b200post_k2pow.h).
#include <algorithm>
#include <atomic>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b200post_k2pow.h"
#include "engine.h"
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

// One window of the prover's search: pows [next, next + per) of every group in `groups`, in one device call.  hit[i] =
// the smallest valid pow of groups[i] in the window, or B200POST_K2POW_NOT_FOUND.
int search_window(RandomxEngine *e, const std::string &key, const b200post_k2pow_params *p, const std::vector<uint32_t> &groups,
                  uint64_t next, uint64_t per, std::vector<uint8_t> &in, std::vector<uint8_t> &out, std::vector<uint64_t> &hit) {
    const size_t n = groups.size() * per;
    in.resize(n * 48); out.resize(n * 32);
    for (size_t gi = 0; gi < groups.size(); gi++)
        for (uint64_t k = 0; k < per; k++) {
            uint8_t *d = &in[(gi * per + k) * 48];
            const uint64_t pow = next + k;
            for (int b = 0; b < 7; b++) d[b] = (uint8_t)(pow >> (8 * b));
            d[7] = (uint8_t)groups[gi];
            memcpy(d + 8, p->challenge8, 8);
            memcpy(d + 16, p->node_id, 32);
        }
    const int rc = e->hash_inputs(key, in.data(), 48, n, out.data());
    if (rc != B200POST_OK) return rc;
    hit.assign(groups.size(), B200POST_K2POW_NOT_FOUND);
    for (size_t gi = 0; gi < groups.size(); gi++)
        for (uint64_t k = 0; k < per && hit[gi] == B200POST_K2POW_NOT_FOUND; k++)
            if (memcmp(&out[(gi * per + k) * 32], p->difficulty, 32) < 0) hit[gi] = next + k;
    return B200POST_OK;
}

// randomx_engine of every entry in list order; the first failing entry's code (and text) answers
int randomx_engines(const uint32_t *providers, int n, std::vector<RandomxEngine *> *out) {
    out->assign((size_t)n, nullptr);
    for (int i = 0; i < n; i++)
        if (int rc = randomx_engine(providers[i], &(*out)[(size_t)i])) return rc;
    return B200POST_OK;
}

}  // namespace

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
    const std::string key = key_of(p->cache_key, p->cache_key_len);
    uint64_t batch = 0;
    e->batch_size(&batch);
    for (uint32_t g = 0; g < n_groups; g++) pows[g] = B200POST_K2POW_NOT_FOUND;
    if (max_nonces_per_group == 0 || max_nonces_per_group > kNonceSpace) max_nonces_per_group = kNonceSpace;
    std::vector<uint32_t> pending(n_groups);   // absolute group numbers: they are the k2pow input's group byte
    for (uint32_t g = 0; g < n_groups; g++) pending[g] = first_group + g;
    std::vector<uint8_t> in, out;
    std::vector<uint64_t> hit;
    uint64_t next = 0, total = 0;      // every pending group has tried nonces [0, next)
    while (!pending.empty() && next < max_nonces_per_group) {
        if (cancel && *cancel) { set_error("cancelled"); return B200POST_ERR_CANCELLED; }
        // one device batch shared by all groups still searching: `per` consecutive nonces each
        const uint64_t per = std::min<uint64_t>(std::max<uint64_t>(1, batch / pending.size()), max_nonces_per_group - next);
        const int rc = search_window(e, key, p, pending, next, per, in, out, hit);
        if (rc != B200POST_OK) return rc;
        total += pending.size() * per;
        std::vector<uint32_t> still;
        for (size_t gi = 0; gi < pending.size(); gi++)
            if (hit[gi] == B200POST_K2POW_NOT_FOUND) still.push_back(pending[gi]); else pows[pending[gi] - first_group] = hit[gi];
        pending.swap(still);
        next += per;
    }
    if (hashes_done) *hashes_done = total;
    return B200POST_OK;
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
    for (uint32_t g = 0; g < n_groups; g++) pows[g] = B200POST_K2POW_NOT_FOUND;
    const std::string key = key_of(p->cache_key, p->cache_key_len);
    const uint64_t cap = max_nonces_per_group == 0 || max_nonces_per_group > kNonceSpace ? kNonceSpace : max_nonces_per_group;
    // Windows go out in ascending nonce order from one cursor, each to every group without a hit yet.  So every group
    // has been handed out the contiguous nonces [0, cursor at its first reported hit), and once all threads have
    // joined, the smallest hit reported for it is its smallest valid pow.
    std::mutex mu;
    uint64_t next = 0, total = 0;
    std::vector<uint64_t> best(n_groups, B200POST_K2POW_NOT_FOUND);
    std::atomic<bool> stop{false};
    const int rc = fan_out((size_t)n_providers, [&](size_t i) {
        uint64_t batch = 0;
        eng[i]->batch_size(&batch);
        std::vector<uint8_t> in, out;
        std::vector<uint64_t> hit;
        std::vector<uint32_t> groups;
        int r = B200POST_OK;
        while (!stop) {
            if (cancel && *cancel) { set_error("cancelled"); r = B200POST_ERR_CANCELLED; break; }
            uint64_t lo, per;
            {
                std::lock_guard<std::mutex> lk(mu);
                groups.clear();
                for (uint32_t g = 0; g < n_groups; g++) if (best[g] == B200POST_K2POW_NOT_FOUND) groups.push_back(first_group + g);
                if (groups.empty() || next >= cap) break;
                // one device batch: `per` consecutive nonces for each group still searching, as on one device
                per = std::min<uint64_t>(std::max<uint64_t>(1, batch / groups.size()), cap - next);
                lo = next;
                next += per;
            }
            if ((r = search_window(eng[i], key, p, groups, lo, per, in, out, hit)) != B200POST_OK) break;
            std::lock_guard<std::mutex> lk(mu);
            total += groups.size() * per;
            for (size_t gi = 0; gi < groups.size(); gi++) best[groups[gi] - first_group] = std::min(best[groups[gi] - first_group], hit[gi]);
        }
        if (r != B200POST_OK) stop = true;
        return r;
    });
    if (hashes_done) *hashes_done = total;
    if (rc) return rc;
    for (uint32_t g = 0; g < n_groups; g++) pows[g] = best[g];
    return B200POST_OK;
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
