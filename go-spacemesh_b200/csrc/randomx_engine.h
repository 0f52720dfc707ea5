// randomx_engine.h — host runtime of the k2pow (RandomX) engine: per-device dataset residency, batch buffers, the launch
// sequence of one batch.  C++ for the same reason as engine.h (the reference's host side is compiled Go; no Go here).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <functional>
#include <mutex>
#include <string>
#include <vector>

#include "cuda_util.h"
#include "randomx_kernels.cuh"

namespace b200post {

class RandomxEngine {
public:
    explicit RandomxEngine(int device);
    ~RandomxEngine();
    RandomxEngine(const RandomxEngine &) = delete;

    int prepare(const std::string &key);
    int hash_inputs(const std::string &key, const uint8_t *inputs, size_t input_len, size_t n, uint8_t *out32);
    // hashes != nullptr: every hash of the range is returned (count x 32).  difficulty != nullptr: search semantics.
    int k2pow(const std::string &key, const rx::K2powTemplate &tmpl, const uint8_t *difficulty, uint64_t start, uint64_t count,
              uint8_t *hashes, uint64_t *found, uint64_t *done, const volatile int *cancel, uint64_t batch_stride = 0,
              const volatile int *peer_hit = nullptr);
    // One device batch of the job search (k2pow_jobs.h): the job table and the batch's segments go to the device, then
    // seeds, the RandomX chain and the compare; hit[s] = the lowest offset into segment s whose hash is below its job's
    // difficulty, or 0xffffffff.  A batch larger than the buffers HBM allowed runs in several launches.  Adds to the
    // timing of last_timing() instead of replacing it (reset_timing() starts a search).
    int search_segments(const std::string &key, const K2powJob *jobs, size_t n_jobs, const JobSegment *segs, size_t n_segs,
                        uint32_t *hit);
    void reset_timing();
    int batch_size(uint64_t *vms);
    // dataset items [first_item, first_item + count) of `key` to host memory (64 bytes each; the range is checked by the caller)
    int dataset_read(const std::string &key, uint64_t first_item, uint64_t count, uint64_t *out);
    void last_timing(double *total_ms, double *vm_ms, uint64_t *hashes, uint64_t *vm_launches);
    // frees the dataset and the batch buffers (~14 GiB); the next call rebuilds them
    void release();

private:
    int ensure_dataset(const std::string &key);
    int ensure_batch(uint32_t want);
    void release_batch();
    // runs seeds..finalize for the n VMs whose seeds are already written
    int run_chain(uint32_t n);
    uint32_t desired_batch() const;

    int dev_;
    cudaDeviceProp prop_{};
    std::mutex mu_;
    Stream stream_;
    bool tables_ = false;
    std::string key_;                       // key of the resident dataset ("" = none)
    DeviceBuffer<uint64_t> d_dataset_;
    rx::BatchBuffers buf_;
    uint32_t cap_ = 0;
    DeviceBuffer<uint8_t> d_inputs_;
    DeviceBuffer<uint8_t> d_diff_;
    DeviceBuffer<uint32_t> d_found_;
    DeviceBuffer<K2powJob> d_jobs_;         // the job search's tables and hit slots
    DeviceBuffer<JobSegment> d_segs_;
    DeviceBuffer<uint32_t> d_hit_;
    PinnedBuffer<uint8_t> h_stage_;   // hashes coming back
    Event ev_[4];
    double total_ms_ = 0, vm_ms_ = 0;
    uint64_t hashes_ = 0, vm_launches_ = 0;
};

RandomxEngine *randomx_engine_for(uint32_t provider);
// randomx_engine_for as a B200POST_* code, as device_engine (engine.h) does for the label engine
int randomx_engine(uint32_t provider, RandomxEngine **e);
void randomx_shutdown_all();

// release() of the engine on `device`, if one was created: its HBM goes back to the device, the engine stays usable
void randomx_release(int device);
// randomx_engine of every entry in list order; the first failing entry's code (and text) answers
int randomx_engines(const uint32_t *providers, int n, std::vector<RandomxEngine *> *out);

// The k2pow job search (b200post_k2pow_search_jobs) on `eng` (one host thread per entry, the calling thread alone for
// one): windows of one JobSchedule over pows [0, cap), each run as device batches on the engine that took it.
// on_final(j, pow) is called, under the schedule's lock, as soon as job j's pow is final.  pows[j] = job j's smallest valid
// pow below the cap or B200POST_K2POW_NOT_FOUND; after an error only final pows are given.  The first failing entry's
// status (list order) is returned once every thread has joined.
int k2pow_search_jobs(const std::vector<RandomxEngine *> &eng, const std::string &key, const std::vector<K2powJob> &jobs, uint64_t cap,
                      uint64_t *pows, uint64_t *hashes_done, const volatile int *cancel,
                      const std::function<void(uint32_t, uint64_t)> &on_final = nullptr);

}  // namespace b200post
