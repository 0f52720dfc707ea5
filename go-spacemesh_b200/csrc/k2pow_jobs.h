// k2pow_jobs.h — the schedule of the k2pow job search (b200post_k2pow_search_jobs), in plain C++ so that it runs, and is
// tested, without a device.
//
// A job is one k2pow: (node_id, challenge[0:8], nonce group, difficulty).  Windows of `per` consecutive nonces go out
// from one cursor in ascending order, each to every job that has no hit yet, and `per` is chosen so that a window fills
// one device batch (batch / pending jobs, at least 1).  A window wider than a batch runs as several batches.  So every
// job has been handed out the contiguous nonces [0, cursor at its first reported hit), and its pow is final (its
// smallest valid pow) once every window below its lowest hit has finished.
#pragma once
#include <cstddef>
#include <cstdint>
#include <map>
#include <vector>

namespace b200post {

// Device layout of one job: the k2pow input's bytes 7..47 (nonce group || challenge[0:8] || node_id) and the
// difficulty, 32 bytes big-endian.
struct K2powJob {
    uint8_t tail[41];
    uint8_t difficulty[32];
};

// Device layout of one segment of a batch: VMs [off, off + cnt) hash job `job` at pows first_pow, first_pow + 1, ...
// A batch's segments are in ascending `off` and cover its VMs without a gap.
struct JobSegment {
    uint32_t off, cnt, job, pad;
    uint64_t first_pow;
};

class JobSchedule {
public:
    static constexpr uint64_t kNotFound = UINT64_MAX;

    struct Window {
        uint64_t id = 0, lo = 0, per = 0;
        std::vector<uint32_t> jobs;   // ascending job numbers
    };

    // n_jobs jobs, each searched over the pows [0, cap) (cap 0 or above 2^56: the whole 56-bit nonce space)
    JobSchedule(size_t n_jobs, uint64_t cap);

    // The next window for a device of `batch` VMs, or false when every job has a hit or the cursor has reached the cap.
    bool take(uint64_t batch, Window *w);
    // The window's device batches: its VMs (job i of the window takes VMs [i * per, (i + 1) * per)) in runs of at most
    // `batch`, each as its segments.
    static std::vector<std::vector<JobSegment>> batches(const Window &w, uint64_t batch);
    // Ends window w: hits[i] is the smallest valid pow of w.jobs[i] in the window, or kNotFound.  Returns the jobs whose
    // pow became final, ascending.
    std::vector<uint32_t> finish(const Window &w, const std::vector<uint64_t> &hits);
    // Jobs that became final without a window ending (the cursor reached the cap), ascending; each is returned once,
    // by this or by finish().
    std::vector<uint32_t> settle();

    uint64_t pow(size_t j) const { return best_[j]; }   // the lowest hit reported so far
    bool final(size_t j) const { return final_[j]; }
    uint64_t hashes() const { return hashes_; }          // sum over the windows handed out of jobs x per

private:
    bool is_final(uint32_t j) const;
    std::vector<uint32_t> newly_final(const std::vector<uint32_t> &candidates);

    uint64_t cap_, next_ = 0, hashes_ = 0, ids_ = 0;
    std::vector<uint64_t> best_;
    std::vector<bool> final_;
    std::map<uint64_t, Window> inflight_;
};

}  // namespace b200post
