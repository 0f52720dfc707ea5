// Drives csrc/k2pow_jobs.cpp (the job search's schedule) without a device, for tests/test_prove_many_host.py: `devices`
// simulated devices take windows and finish them in a seeded random order; a job's valid pows are given as sorted lists.
#include <cstdint>
#include <random>
#include <vector>

#include "../go-spacemesh_b200/csrc/k2pow_jobs.h"

using namespace b200post;

extern "C" int emul_search(uint32_t n_jobs, const uint64_t *valid, const uint32_t *first_valid, uint64_t cap, uint64_t batch,
                           uint32_t devices, uint32_t seed, uint64_t *pows, uint64_t *final_pow, uint64_t *hashes,
                           uint64_t *n_batches) {
    JobSchedule sched(n_jobs, cap);
    std::mt19937_64 rng(seed);
    std::vector<JobSchedule::Window> held(devices);
    std::vector<bool> busy(devices, false), ended(devices, false);
    *n_batches = 0;
    const auto mark = [&](const std::vector<uint32_t> &done) -> int {
        for (uint32_t j : done) {
            if (final_pow[j] != UINT64_MAX - 1) return 1;   // final twice
            final_pow[j] = sched.pow(j);
        }
        return 0;
    };
    for (uint32_t j = 0; j < n_jobs; j++) final_pow[j] = UINT64_MAX - 1;
    for (;;) {
        bool any = false;
        for (uint32_t d = 0; d < devices; d++) any |= busy[d] || !ended[d];
        if (!any) break;
        const uint32_t d = (uint32_t)(rng() % devices);
        if (ended[d] && !busy[d]) continue;
        if (!busy[d]) {
            if (sched.take(batch, &held[d])) busy[d] = true;
            else { ended[d] = true; if (mark(sched.settle())) return 1; }
            continue;
        }
        const JobSchedule::Window &w = held[d];
        std::vector<uint64_t> hits(w.jobs.size(), JobSchedule::kNotFound);
        for (const auto &segs : JobSchedule::batches(w, batch)) {
            (*n_batches)++;
            uint64_t vms = 0;
            for (const JobSegment &s : segs) {
                if (s.off != vms) return 2;   // segments must tile the batch
                vms += s.cnt;
                size_t k = 0;
                while (w.jobs[k] != s.job) k++;
                for (uint32_t i = first_valid[s.job]; i < first_valid[s.job + 1]; i++)
                    if (valid[i] >= s.first_pow && valid[i] < s.first_pow + s.cnt) { if (valid[i] < hits[k]) hits[k] = valid[i]; break; }
            }
            if (vms > batch) return 3;
        }
        if (mark(sched.finish(w, hits))) return 1;
        busy[d] = false;
    }
    for (uint32_t j = 0; j < n_jobs; j++) pows[j] = sched.final(j) ? sched.pow(j) : UINT64_MAX - 1;
    *hashes = sched.hashes();
    return 0;
}
