// engine.h — host runtime of the POST label engine: per-device scratch, layer scheduling,
// double-buffered staging.  C++ because the reference's host side for this path is compiled code
// (Go: activation/post.go PostSetupManager, activation/post_verifier.go); the Go toolchain is absent
// in this image (INTEGRATION.md shows the cgo binding that sits on top of the C ABI).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <deque>
#include <functional>
#include <mutex>
#include <string>
#include <vector>

#include "label_kernels.cuh"
#include "cuda_util.h"
#include "rider_plan.h"

namespace b200post {

struct Options {
    std::atomic<int64_t> romix_variant{ROMIX_PHASED};
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
// outcome of a compare job: how many recomputed labels differ from the expected bytes, and the lowest
// kMaxReported of their positions in job order (ascending), whatever the layer shape
struct CompareResult {
    static constexpr size_t kMaxReported = 64;
    uint64_t mismatches = 0;
    std::vector<uint64_t> first;
};

void set_error(const std::string &msg);
const char *last_error();
int fail(int rc, const std::string &msg);   // set_error(msg), then rc

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
    // path recomputes ~37 labels per identity, so the commitment H2D shrinks by that factor.  out_hi_dev (optional, only
    // with out_dev): device buffer of n_items*16 bytes that gets bytes 16-31 of every label32 (K3w instead of K3).
    // A row index past n_commit is B200POST_ERR_INVALID_ARGUMENT.
    //
    // Riders: a gather-class call (labels_gather, labels_gather_indexed, labels_compare_indexed) that arrives while a
    // range job of the same N runs on this engine does not wait for that job to end.  It queues as a rider, the range
    // job packs queued riders into the free slots of its next layers (FIFO, at most half of each layer, rider_plan.h),
    // and the call returns once its last chunk has retired.  Riders still queued when the range job ends run as ordinary
    // calls; a CUDA error in a shared layer fails every rider in it with the host job's code and text.  A rider does not
    // look at its cancel flag once queued.
    int labels_gather_indexed(size_t n_items, size_t n_commit, const uint8_t *commitments, const uint32_t *commit_index,
                              const uint64_t *indices, uint64_t N, uint8_t *out_host, uint8_t *out_dev,
                              uint8_t *out_hi_dev = nullptr);
    // compare jobs (K3c): recompute labels and compare them with expect_host (16 bytes per item, in job order) instead of
    // returning them.  Range form: labels [start, start + count), VRF scan as in labels_range.  Indexed form: the labels
    // at `indices` under one commitment.  *cmp is reset by the call; on CANCELLED it holds what was compared so far.
    int labels_compare_range(const uint8_t commitment[32], uint64_t N, uint64_t start, uint64_t count, const uint8_t *expect_host,
                             const uint8_t *vrf_difficulty, VrfResult *vrf, CompareResult *cmp, const volatile int *cancel);
    int labels_compare_indexed(const uint8_t commitment[32], size_t n_items, const uint64_t *indices, uint64_t N,
                               const uint8_t *expect_host, CompareResult *cmp, const volatile int *cancel);
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
        const uint8_t *commit_table = nullptr;  // indexed gather: the call's n_commit x 32 rows; compare-indexed: its one
                                                // commitment (host; riders stage from it)
        const uint64_t *indices = nullptr;      // gather: n (host)
        const uint32_t *commit_index = nullptr; // indexed gather: per-item row of the call-level commitment table
                                                // (gather with neither: every item uses the call's one commitment)
        const uint8_t *expect_host = nullptr;   // compare job: expected labels, 16 bytes per item in job order
        CompareResult *cmp = nullptr;
        VrfResult *vrf = nullptr;
        uint64_t start = 0, total = 0, N = 0;
        uint8_t *out_host = nullptr, *out_dev = nullptr;
        uint8_t *out_hi_dev = nullptr;          // gather: bytes 16-31 of each label32 (device, with out_dev; K3w)
        const uint32_t *d_diff = nullptr;
        const volatile int *cancel = nullptr;
        // the commitment of item i of a gather-class job
        const uint8_t *row(uint64_t i) const {
            return commit_index ? commit_table + 32 * (size_t)commit_index[i] : commitments ? commitments + 32 * i : commit_table;
        }
    };
    // A gather-class call queued on a running range job (see labels_gather_indexed).  The caller owns it and blocks
    // until `done` (result in rc / err) or `released` (the range job ended first: items [retired, items) are left).
    struct Rider {
        RiderLoad load;
        uint64_t retired = 0;            // items whose layers have retired
        const Job *job = nullptr;
        bool done = false, released = false;
        int rc = 0;
        std::string err;
    };
    // Everything one layer parity owns: its slot buffers, events and in-flight bookkeeping.
    struct Layer {
        DeviceBuffer<uint4> X;
        DeviceBuffer<uint8_t> d_out, d_commit;
        PinnedBuffer<uint8_t> h_out, h_commit;          // pinned staging of outputs and gather inputs
        DeviceBuffer<uint64_t> d_idx;
        PinnedBuffer<uint64_t> h_idx;
        DeviceBuffer<uint32_t> d_cidx;                  // indexed gather: per-item commitment rows
        PinnedBuffer<uint32_t> h_cidx;
        // compare jobs: expected labels (pinned staging -> device, on copy_stream_), K3c's mismatch bitmap and count
        DeviceBuffer<uint8_t> d_exp;
        PinnedBuffer<uint8_t> h_exp;
        DeviceBuffer<uint32_t> d_bits, d_cnt;
        PinnedBuffer<uint32_t> h_cnt;
        Event ev_done;        // layer outputs are in h_out
        Event ev_k3;          // K3 of the layer has written d_out (the copy stream waits on it)
        Event ev_in;          // layer inputs have left h_commit / h_idx / h_cidx
        Event ev_exp;         // the expected slice of the layer is on the device
        Event ev_k2a, ev_k2b; // bracket the ROMix launch (timed)
        bool in_pending = false, k2_pending = false;
        double k2_labels = 0;
        // the layer being staged: its segments (range labels or a gather's items, then rider chunks) and each chunk's rider
        LayerPlan plan;
        std::vector<Rider *> chunk_rider;
        // the finished layer retire() waits for (the pipelined loop stages this parity again before retiring it)
        struct Pending { LayerPlan plan; std::vector<Rider *> riders; bool live = false; } pend;
        int allocate(uint32_t slots);   // (re)creates every buffer and event for `slots` slots
    };
    // mu_, held for the scope (locked = already taken by try_lock); its release wakes gathers waiting in call()
    struct Hold {
        explicit Hold(DeviceEngine &e, bool locked = false);
        ~Hold();
        DeviceEngine &e_;
    };
    // the label calls: a gather-class call rides a range job when it can (ride()), else it holds the engine for run_call()
    int call(Job &job, const std::function<int()> &setup);
    // the shared body of the label calls, mu_ held: scratch, `setup` (per-call uploads), the timed job, metrics
    int run_call(Job &job, const std::function<int()> &setup);
    // true when the call rode a range job (*rc: its result, leftovers included); false: not now
    bool ride(Job &job, const std::function<int()> &setup, int *rc);
    // the range job in run_job has ended with `status`: fail the riders of its failed layers, release the rest
    void end_hosting(int status);
    // l.plan / l.chunk_rider = the next layer of `job` from its item range_off on: at most S of its labels, plus the
    // queued riders when the job hosts them
    void next_layer(const Job &job, uint64_t range_off, uint64_t S, bool host, Layer &l);
    int ensure(uint64_t N, uint64_t want_slots);   // (re)allocates scratch; sets wave_slots_
    int run_job(const Job &job);
    int range_call(Job &job, const uint8_t commitment[32], const uint8_t *vrf_difficulty);
    int upload_commitment(const uint8_t commitment[32]);
    // b = buffer parity of the layer (layer index + parity offset of the call)
    // l.plan says which labels: the range segment (or a gather's items) and the rider chunks
    int stage_layer(const Job &job, int b, LabelJob *lj);          // inputs + K1
    int finish_layer(const Job &job, int b, const LabelJob &lj);   // K3 (+K4) + D2H + event
    int retire(const Job &job, int buf);
    void harvest(int buf);
    void quiesce();   // after an error: drain the stream, drop in-flight bookkeeping

    int dev_;
    cudaDeviceProp prop_{};
    std::mutex mu_;
    // riders: queued gathers and whether a range job (of scrypt-N host_N_) takes them now
    std::mutex rider_mu_;
    std::condition_variable rider_cv_;
    std::deque<Rider *> riders_;
    bool hosting_ = false;
    uint64_t host_N_ = 0;
    uint64_t release_gen_ = 0;             // releases of mu_ so far
    Stream stream_;
    Stream copy_stream_;                   // D2H of finished labels, off the kernels' stream
    // scratch
    DeviceBuffer<uint8_t> V_raw_;
    uint4 *V_ = nullptr;                   // aligned view into V_raw_
    size_t v_bytes_ = 0, v_align_ = 0;
    uint32_t alloc_slots_ = 0;             // capacity of the per-slot buffers of layer_, in labels
    uint32_t wave_slots_ = 0;              // resident slots (ROMix threads with their scratch) for the current (N, options)
    uint32_t layer_labels_ = 0;            // labels per layer: wave_slots_, or twice that for ROMIX_PHASED
    Layer layer_[2];                       // per-layer state, double-buffered by layer parity
    DeviceBuffer<uint32_t> d_range_commit_;   // the commitment of the current call (32 bytes)
    DeviceBuffer<uint8_t> d_ctab_;            // indexed gather: call-level commitment table
    DeviceBuffer<uint32_t> d_diff_;
    DeviceBuffer<VrfCandidate> d_cta_cand_, d_running_;
    PinnedBuffer<VrfCandidate> h_running_;
    Event ev_call_[2];
    double last_call_ms_ = 0;
    Event ev_timer_[2];
    double romix_ms_ = 0, romix_labels_ = 0;
    uint64_t romix_launches_ = 0;
    // Speculative continuation (pipelined range jobs): the launch that mixes the last layer of a call also fills
    // the first layer of the range that would follow it (start + count ...).  If the next call is exactly that
    // range (same commitment and N), it starts with that layer already filled, so back-to-back initialize()
    // batches run as one uninterrupted software pipeline instead of draining after every call.  ensure() drops it
    // whenever it reallocates the scratch or changes the layer size.
    struct Speculation {
        bool valid = false;
        uint8_t commitment[32] = {0};
        uint64_t N = 0, next_start = 0;
        int parity = 0;
    } spec_;
    uint8_t cur_commitment_[32] = {0};
    // current tuning
    int variant_ = ROMIX_PIPELINED, mw_ = 0, tpb_ = 512, dr_unroll_ = 4;
};

// registry: lazily created engine per CUDA ordinal (nullptr + error text if the device is unusable)
DeviceEngine *engine_for(uint32_t provider);
// engine_for as a B200POST_* code: B200POST_ERR_UNSUPPORTED for the CPU id (no CPU path), B200POST_ERR_NO_DEVICE for an
// id that names no device.  e / out (optional) get the engines.  A list answers with its first failing entry's code.
int device_engine(uint32_t provider, DeviceEngine **e = nullptr);
int device_engines(const uint32_t *providers, int n, std::vector<DeviceEngine *> *out = nullptr);
int device_count();
// The CUDA ordinals a provider id names at a host entry point: every device for B200POST_PROVIDER_ALL, else the id.
// B200POST_ERR_UNSUPPORTED for the CPU id, B200POST_ERR_NO_DEVICE when the machine has no device; an ordinal past the
// last device is left to engine_for.
int provider_devices(int64_t provider_id, std::vector<uint32_t> *devs);
void shutdown_all();

// Runs part(0) .. part(parts - 1) on one thread each and returns once all have ended: B200POST_OK, or the code of the
// first failing part in list order, whose error text (thread-local, so copied out as its thread ends) is then this
// thread's.
int fan_out(size_t parts, const std::function<int(size_t)> &part);

// The label32 at `index` (one label, recomputed on e); all-ones is a label32 like any other
int label32_at(DeviceEngine *e, const uint8_t commitment[32], uint64_t N, uint64_t index, uint8_t out[32]);

}  // namespace b200post
