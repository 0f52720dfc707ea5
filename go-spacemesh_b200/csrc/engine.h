// engine.h — host runtime of the POST label engine: per-device scratch, layer scheduling,
// double-buffered staging.  C++ because the reference's host side for this path is compiled code
// (Go: activation/post.go PostSetupManager, activation/post_verifier.go); the Go toolchain is absent
// in this image (INTEGRATION.md shows the cgo binding that sits on top of the C ABI).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <memory>
#include <mutex>
#include <string>

#include "label_kernels.cuh"

namespace b200post {

struct Options {
    std::atomic<int64_t> romix_variant{ROMIX_PIPELINED};
    std::atomic<int64_t> rotate_mask{0};
    std::atomic<int64_t> tpb{512};             // CTA size; the pipelined kernel takes smaller CTAs when HBM cannot give every SM one of this size
    std::atomic<int64_t> dr_unroll{4};         // pipelined kernel: ChaCha double-rounds unrolled (4) or rolled (1)
    std::atomic<int64_t> ctas_per_sm{0};       // 0 = occupancy maximum
    std::atomic<int64_t> max_scratch_mib{0};   // 0 = 95 % of free HBM
    std::atomic<int64_t> speculate_next{1};    // pipelined range jobs of >= 4 layers pre-fill the next range's first layer
    std::atomic<int64_t> lowlat_max_labels{4096};   // jobs of at most this many labels take the low-latency ROMix kernel (0 = never)
    std::atomic<int64_t> rx_vms_per_sm{0};     // k2pow: RandomX VMs (2 MiB scratchpads) resident per SM in one batch; 0 = the mode's default
    std::atomic<int64_t> rx_vm_mode{1};        // k2pow VM kernel variant: 0 = 32 VMs/SM (<= 64 regs), 1 = 48 VMs/SM (default), 2 = 64 VMs/SM
    std::atomic<int64_t> debug_corrupt_next_batch{0};   // tests: flip one bit in the next init batch before the self-check (one-shot)
    std::atomic<int64_t> debug_corrupt_check_all{0};    // tests: make the self-check look at the label the injected fault hits
    std::atomic<int64_t> debug_skip_phase{0};  // diagnostics only (classic variants): bit0 skip fill, bit1 skip mix
};
Options &options();

extern std::atomic<uint64_t> g_launches;

struct VrfResult { bool found = false; uint64_t index = 0; uint8_t label32[32] = {0}; };

void set_error(const std::string &msg);
const char *last_error();

class DeviceEngine {
public:
    explicit DeviceEngine(int device);
    ~DeviceEngine();
    DeviceEngine(const DeviceEngine &) = delete;

    // out_host / out_dev: at most one non-null (both null = discard).  Returns a B200POST_* code.
    int labels_range(const uint8_t commitment[32], uint64_t N, uint64_t start, uint64_t count, uint8_t *out_host,
                     uint8_t *out_dev, const uint8_t *vrf_difficulty, VrfResult *vrf, const volatile int *cancel);
    // out_dev (optional): device buffer of n_items*16 bytes on this device; the labels then never leave HBM
    int labels_gather(size_t n_items, const uint8_t *commitments, const uint64_t *indices, uint64_t N, uint8_t *out_host,
                      uint8_t *out_dev = nullptr);
    // same with the commitments given once (n_commit x 32 bytes) and a per-item row index into them: the verify
    // path recomputes ~37 labels per identity, so the commitment H2D shrinks by that factor
    int labels_gather_indexed(size_t n_items, size_t n_commit, const uint8_t *commitments, const uint32_t *commit_index,
                              const uint64_t *indices, uint64_t N, uint8_t *out_host, uint8_t *out_dev);
    // accumulated ROMix kernel device time, launches, and label-equivalents processed by those launches
    void romix_time(double *ms_total, uint64_t *launches, double *labels, bool reset);
    // device time (CUDA events on the engine's stream) of the last labels_range / labels_gather call
    double last_call_ms();
    // stopwatch on the engine's own stream: mark(0) ... mark(1), then elapsed (CUDA events; includes gaps between calls)
    int timer_mark(int which);
    double timer_elapsed_ms();
    // labels one layer (wave) holds for scrypt-N under the current options; 0 + error text on failure
    uint32_t wave_slots(uint64_t N);
    int device() const { return dev_; }
    const cudaDeviceProp &prop() const { return prop_; }

private:
    struct Job {
        bool gather = false;
        const uint8_t *commitments = nullptr;   // gather: n x 32 (host)
        const uint64_t *indices = nullptr;      // gather: n (host)
        const uint32_t *commit_index = nullptr; // indexed gather: per-item row of the call-level commitment table
        uint64_t start = 0, total = 0, N = 0;
        uint8_t *out_host = nullptr, *out_dev = nullptr;
        const uint32_t *d_diff = nullptr;
        const volatile int *cancel = nullptr;
    };
    int ensure(uint64_t N, uint64_t want_slots);   // (re)allocates scratch; sets wave_slots_
    void release();
    int run_job(const Job &job);
    // b = buffer parity of the layer (layer index + parity offset of the call)
    int stage_layer(const Job &job, uint64_t layer, int b, uint32_t n_valid, LabelJob *lj);          // inputs + K1
    int finish_layer(const Job &job, uint64_t layer, int b, uint32_t n_valid, const LabelJob &lj);   // K3 (+K4) + D2H + event
    int retire(const Job &job, int buf);
    void harvest(int buf);
    void quiesce();   // after an error: drain the stream, drop in-flight bookkeeping

    int dev_;
    cudaDeviceProp prop_{};
    std::mutex mu_;
    cudaStream_t stream_ = nullptr;
    // scratch
    uint4 *V_ = nullptr;         // aligned view into V_raw_
    void *V_raw_ = nullptr;
    size_t v_bytes_ = 0, v_align_ = 0;
    uint32_t alloc_slots_ = 0;   // capacity of the per-slot buffers below
    uint32_t wave_slots_ = 0;    // slots per layer for the current (N, options)
    // per-layer state, double-buffered by layer parity
    uint4 *X_[2] = {nullptr, nullptr};
    uint8_t *d_out_[2] = {nullptr, nullptr};
    uint8_t *h_out_[2] = {nullptr, nullptr};       // pinned
    uint8_t *d_commit_[2] = {nullptr, nullptr};
    uint64_t *d_idx_[2] = {nullptr, nullptr};
    uint8_t *h_commit_[2] = {nullptr, nullptr};    // pinned staging for gather inputs
    uint64_t *h_idx_[2] = {nullptr, nullptr};
    uint32_t *d_range_commit_ = nullptr;   // the commitment of the current range call (32 bytes)
    uint32_t *d_cidx_[2] = {nullptr, nullptr}, *h_cidx_[2] = {nullptr, nullptr};   // indexed gather: per-item commitment rows
    uint8_t *d_ctab_ = nullptr; size_t ctab_rows_ = 0;   // indexed gather: call-level commitment table
    uint32_t *d_diff_ = nullptr;
    VrfCandidate *d_cta_cand_ = nullptr;
    VrfCandidate *d_running_ = nullptr;
    VrfCandidate *h_running_ = nullptr;            // pinned
    cudaEvent_t ev_done_[2] = {nullptr, nullptr};  // layer outputs are in h_out_[b]
    cudaEvent_t ev_k3_[2] = {nullptr, nullptr};    // K3 of the layer has written d_out_[b] (the copy stream waits on it)
    cudaStream_t copy_stream_ = nullptr;           // D2H of finished labels, off the kernels' stream
    cudaEvent_t ev_in_[2] = {nullptr, nullptr};    // layer inputs have left h_commit_/h_idx_[b]
    bool in_pending_[2] = {false, false};
    cudaEvent_t ev_k2a_[2] = {nullptr, nullptr}, ev_k2b_[2] = {nullptr, nullptr};
    bool k2_pending_[2] = {false, false};
    double k2_labels_[2] = {0, 0};
    struct Pending { uint64_t off; uint32_t n; bool live; } pend_[2] = {{0, 0, false}, {0, 0, false}};
    cudaEvent_t ev_call_[2] = {nullptr, nullptr};
    double last_call_ms_ = 0;
    cudaEvent_t ev_timer_[2] = {nullptr, nullptr};
    double romix_ms_ = 0, romix_labels_ = 0;
    uint64_t romix_launches_ = 0;
    // Speculative continuation (pipelined range jobs): the launch that mixes the last layer of a call also fills
    // the first layer of the range that would follow it (start + count ...).  If the next call is exactly that
    // range (same commitment, N, buffers), it starts with that layer already filled, so back-to-back initialize()
    // batches run as one uninterrupted software pipeline instead of draining after every call.
    struct Speculation {
        bool valid = false;
        uint8_t commitment[32] = {0};
        uint64_t N = 0, next_start = 0;
        int parity = 0;
        uint32_t slots = 0, alloc_slots = 0;
        const void *V = nullptr;
    } spec_;
    uint8_t cur_commitment_[32] = {0};
    // current tuning
    int variant_ = ROMIX_PIPELINED, mw_ = 0, tpb_ = 512, dr_unroll_ = 4;
};

// registry: lazily created engine per CUDA ordinal (nullptr + error text if the device is unusable)
DeviceEngine *engine_for(uint32_t provider);
int device_count();
void shutdown_all();

}  // namespace b200post
