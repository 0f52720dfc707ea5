// randomx_engine.h — host runtime of the k2pow (RandomX) engine: per-device dataset residency, batch buffers, the launch
// sequence of one batch.  C++ for the same reason as engine.h (the reference's host side is compiled Go; no Go here).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <mutex>
#include <string>

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
    PinnedBuffer<uint8_t> h_stage_;   // hashes coming back
    Event ev_[4];
    double total_ms_ = 0, vm_ms_ = 0;
    uint64_t hashes_ = 0, vm_launches_ = 0;
};

RandomxEngine *randomx_engine_for(uint32_t provider);
void randomx_shutdown_all();
// release() of the engine on `device`, if one was created: its HBM goes back to the device, the engine stays usable
void randomx_release(int device);

}  // namespace b200post
