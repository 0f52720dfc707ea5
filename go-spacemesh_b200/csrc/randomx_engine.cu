// randomx_engine.cu — see randomx_engine.h.
#include "randomx_engine.h"

#include <algorithm>
#include <cstring>
#include <map>
#include <memory>
#include <vector>

#include "../../include/b200post.h"
#include "engine.h"

namespace b200post {

RandomxEngine::RandomxEngine(int device) : dev_(device) {
    cudaGetDeviceProperties(&prop_, device);
}

RandomxEngine::~RandomxEngine() {
    // the other members free themselves after this body, on this device and with no work of the engine in flight
    cudaSetDevice(dev_);
    if (stream_.get()) cudaStreamSynchronize(stream_.get());
    release_batch();
}

void RandomxEngine::release_batch() {
    cudaFree(buf_.scratchpads); cudaFree(buf_.hot); cudaFree(buf_.program); cudaFree(buf_.rcp); cudaFree(buf_.seed); cudaFree(buf_.regfile);
    cudaFree(buf_.config); cudaFree(buf_.fprc); cudaFree(buf_.hashes);
    buf_ = rx::BatchBuffers{};
    cap_ = 0;
}

uint32_t RandomxEngine::desired_batch() const {
    int64_t per_sm = options().rx_vms_per_sm.load();
    if (per_sm <= 0) { const int64_t m = options().rx_vm_mode.load(); per_sm = m == 0 ? 32 : m == 1 ? 48 : m == 2 ? 64 : 40; }   // = resident warps per SM of the variant
    return (uint32_t)std::min<int64_t>((int64_t)prop_.multiProcessorCount * per_sm, 1 << 20);
}

int RandomxEngine::ensure_dataset(const std::string &key) {
    CUDA_TRY(cudaSetDevice(dev_));
    if (!stream_.get()) {
        CUDA_TRY(stream_.create(cudaStreamNonBlocking));
        for (Event &e : ev_) CUDA_TRY(e.create(cudaEventDefault));
        CUDA_TRY(d_diff_.resize(32));
        CUDA_TRY(d_found_.resize(1));
    }
    if (!tables_) { CUDA_TRY(rx::upload_tables()); tables_ = true; }
    if (d_dataset_.get() && key_ == key) return B200POST_OK;
    // host: Argon2d cache + the 8 SuperscalarHash programs (sequential by construction, ~0.7 s)
    rx::CacheImage img;
    rx::build_cache(key.data(), key.size(), img);
    std::vector<rx::SsOp> flat;
    rx::SuperscalarImage ss;
    for (uint32_t i = 0; i < rx::kCacheAccesses; i++) {
        ss.first[i] = (uint32_t)flat.size();
        ss.address_reg[i] = img.programs[i].address_reg;
        flat.insert(flat.end(), img.programs[i].ops.begin(), img.programs[i].ops.end());
    }
    ss.first[rx::kCacheAccesses] = (uint32_t)flat.size();
    DeviceBuffer<uint64_t> d_cache;
    DeviceBuffer<rx::SsOp> d_ops;
    key_.clear();
    if (!d_dataset_.get()) CUDA_TRY(d_dataset_.resize(rx::kDatasetItems * 8));
    CUDA_TRY(d_cache.resize(img.memory.size()));
    CUDA_TRY(d_ops.resize(flat.size()));
    CUDA_TRY(cudaMemcpyAsync(d_cache.get(), img.memory.data(), img.memory.size() * 8, cudaMemcpyHostToDevice, stream_.get()));
    CUDA_TRY(cudaMemcpyAsync(d_ops.get(), flat.data(), flat.size() * sizeof(rx::SsOp), cudaMemcpyHostToDevice, stream_.get()));
    ss.ops = d_ops.get();
    CUDA_TRY(rx::launch_dataset(d_cache.get(), ss, d_dataset_.get(), 0, rx::kDatasetItems, stream_.get()));
    g_launches.fetch_add(1);
    CUDA_TRY(cudaStreamSynchronize(stream_.get()));
    key_ = key;
    return B200POST_OK;
}

int RandomxEngine::ensure_batch(uint32_t want) {
    want = std::max<uint32_t>(32, (want + 31) / 32 * 32);
    if (want <= cap_) return B200POST_OK;
    CUDA_TRY(cudaStreamSynchronize(stream_.get()));
    release_batch();
    // shrink until it fits next to whatever else lives on the device (the label engine's scratch, other datasets)
    for (uint32_t cap = want;; cap = std::max<uint32_t>(32, cap / 2 / 32 * 32)) {
        size_t free_b = 0, total_b = 0;
        CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
        const size_t per_vm = (size_t)rx::kScratchpadL3 + rx::kScratchpadL1 + 256 * 8 + rx::kRcpSlots * 8 + 64 + 256 + 32 + 1 + 32;
        if ((size_t)cap * per_vm + ((size_t)256 << 20) <= free_b) {
            rx::BatchBuffers b;
            b.stride = cap;
            cudaError_t e = cudaMalloc(&b.scratchpads, (size_t)cap * rx::kScratchpadL3);
            if (e == cudaSuccess) e = cudaMalloc(&b.hot, (size_t)cap * rx::kScratchpadL1);
            if (e == cudaSuccess) e = cudaMalloc(&b.program, (size_t)cap * 256 * sizeof(uint2));
            if (e == cudaSuccess) e = cudaMalloc(&b.rcp, (size_t)cap * rx::kRcpSlots * 8);
            if (e == cudaSuccess) e = cudaMalloc(&b.seed, (size_t)cap * 64);
            if (e == cudaSuccess) e = cudaMalloc(&b.regfile, (size_t)cap * 256);
            if (e == cudaSuccess) e = cudaMalloc(&b.config, (size_t)cap * 32);
            if (e == cudaSuccess) e = cudaMalloc(&b.fprc, cap);
            if (e == cudaSuccess) e = cudaMalloc(&b.hashes, (size_t)cap * 32);
            buf_ = b;
            if (e == cudaSuccess) { cap_ = cap; break; }
            cudaGetLastError();
            release_batch();
        }
        if (cap == 32) { set_error("not enough HBM for one warp of RandomX scratchpads (2 MiB each)"); return B200POST_ERR_OUT_OF_MEMORY; }
    }
    // (A persisting-L2 access-policy window over the hot plane was measured twice: 4 361 vs 4 370 H/s with the first
    // warp-per-VM kernel and 6 367 vs 6 377 H/s with the current one, no gain; the L2 set-aside also slowed the label
    // kernels of a following verify batch by a third.  Not used.)
    CUDA_TRY(h_stage_.grow((size_t)cap_ * 32));
    return B200POST_OK;
}

int RandomxEngine::run_chain(uint32_t n) {
    const int vm_mode = (int)options().rx_vm_mode.load();
    CUDA_TRY(rx::launch_fill_scratchpads(buf_, n, stream_.get()));
    for (int p = 0; p < rx::kProgramCount; p++) {
        CUDA_TRY(rx::launch_program(buf_, n, p == 0, stream_.get()));
        CUDA_TRY(cudaEventRecord(ev_[2].get(), stream_.get()));
        CUDA_TRY(rx::launch_execute(buf_, n, d_dataset_.get(), vm_mode, stream_.get()));
        CUDA_TRY(cudaEventRecord(ev_[3].get(), stream_.get()));
        if (p + 1 < rx::kProgramCount) CUDA_TRY(rx::launch_chain_seed(buf_, n, stream_.get()));
        // the VM kernel's own time: events bracket it on the launching stream; summed after the sync below
        CUDA_TRY(cudaEventSynchronize(ev_[3].get()));
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, ev_[2].get(), ev_[3].get()));
        vm_ms_ += ms; vm_launches_++;
    }
    CUDA_TRY(rx::launch_finalize(buf_, n, stream_.get()));
    g_launches.fetch_add(1 + 8 * 2 + 7 + 2);
    return B200POST_OK;
}

int RandomxEngine::prepare(const std::string &key) {
    std::lock_guard<std::mutex> lk(mu_);
    return ensure_dataset(key);
}

int RandomxEngine::batch_size(uint64_t *vms) {
    std::lock_guard<std::mutex> lk(mu_);
    if (vms) *vms = desired_batch();
    return B200POST_OK;
}

int RandomxEngine::dataset_read(const std::string &key, uint64_t first_item, uint64_t count, uint64_t *out) {
    std::lock_guard<std::mutex> lk(mu_);
    const int rc = ensure_dataset(key);
    if (rc != B200POST_OK || count == 0) return rc;
    CUDA_TRY(cudaMemcpyAsync(out, d_dataset_.get() + first_item * 8, count * 64, cudaMemcpyDeviceToHost, stream_.get()));
    CUDA_TRY(cudaStreamSynchronize(stream_.get()));
    return B200POST_OK;
}

void RandomxEngine::last_timing(double *total_ms, double *vm_ms, uint64_t *hashes, uint64_t *vm_launches) {
    std::lock_guard<std::mutex> lk(mu_);
    if (total_ms) *total_ms = total_ms_;
    if (vm_ms) *vm_ms = vm_ms_;
    if (hashes) *hashes = hashes_;
    if (vm_launches) *vm_launches = vm_launches_;
}

void RandomxEngine::release() {
    std::lock_guard<std::mutex> lk(mu_);
    cudaSetDevice(dev_);
    if (stream_.get()) cudaStreamSynchronize(stream_.get());
    release_batch();
    d_dataset_.reset();
    d_inputs_.reset();
    key_.clear();
}

int RandomxEngine::hash_inputs(const std::string &key, const uint8_t *inputs, size_t input_len, size_t n, uint8_t *out32) {
    std::lock_guard<std::mutex> lk(mu_);
    int rc = ensure_dataset(key);
    if (rc != B200POST_OK) return rc;
    total_ms_ = vm_ms_ = 0; hashes_ = vm_launches_ = 0;
    if (n == 0) return B200POST_OK;
    rc = ensure_batch((uint32_t)std::min<size_t>(n, desired_batch()));
    if (rc != B200POST_OK) return rc;
    const size_t need_in = (size_t)cap_ * std::max<size_t>(input_len, 1);
    CUDA_TRY(d_inputs_.grow(need_in));
    const uint32_t batch = std::min<uint32_t>(cap_, desired_batch());
    for (size_t off = 0; off < n; off += batch) {
        const uint32_t m = (uint32_t)std::min<size_t>(batch, n - off);
        CUDA_TRY(cudaEventRecord(ev_[0].get(), stream_.get()));
        if (input_len) CUDA_TRY(cudaMemcpyAsync(d_inputs_.get(), inputs + off * input_len, (size_t)m * input_len, cudaMemcpyHostToDevice, stream_.get()));
        CUDA_TRY(rx::launch_seed_inputs(buf_, m, d_inputs_.get(), (uint32_t)input_len, stream_.get()));
        rc = run_chain(m);
        if (rc != B200POST_OK) return rc;
        CUDA_TRY(cudaMemcpyAsync(h_stage_.get(), buf_.hashes, (size_t)m * 32, cudaMemcpyDeviceToHost, stream_.get()));
        CUDA_TRY(cudaEventRecord(ev_[1].get(), stream_.get()));
        CUDA_TRY(cudaStreamSynchronize(stream_.get()));
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, ev_[0].get(), ev_[1].get()));
        total_ms_ += ms; hashes_ += m;
        memcpy(out32 + off * 32, h_stage_.get(), (size_t)m * 32);
    }
    return B200POST_OK;
}

int RandomxEngine::k2pow(const std::string &key, const rx::K2powTemplate &tmpl, const uint8_t *difficulty, uint64_t start, uint64_t count,
                         uint8_t *hashes, uint64_t *found, uint64_t *done, const volatile int *cancel, uint64_t batch_stride,
                         const volatile int *peer_hit) {
    std::lock_guard<std::mutex> lk(mu_);
    if (found) *found = UINT64_MAX;
    if (done) *done = 0;
    int rc = ensure_dataset(key);
    if (rc != B200POST_OK) return rc;
    total_ms_ = vm_ms_ = 0; hashes_ = vm_launches_ = 0;
    if (count == 0) return B200POST_OK;
    rc = ensure_batch((uint32_t)std::min<uint64_t>(count, desired_batch()));
    if (rc != B200POST_OK) return rc;
    if (difficulty) CUDA_TRY(cudaMemcpyAsync(d_diff_.get(), difficulty, 32, cudaMemcpyHostToDevice, stream_.get()));
    // batch_stride != 0: this device owns batches at start + k * batch_stride (interleaved multi-device search)
    const uint32_t batch = std::min<uint32_t>(cap_, desired_batch());   // cap_ may be left over from a larger setting
    const uint64_t step = batch_stride ? batch_stride : batch;
    for (uint64_t off = 0; off < count; off += step) {
        if (cancel && *cancel) { set_error("cancelled"); return B200POST_ERR_CANCELLED; }
        if (peer_hit && *peer_hit) break;
        const uint32_t m = (uint32_t)std::min<uint64_t>(batch, count - off);
        rx::K2powTemplate t = tmpl;
        t.start = start + off;
        CUDA_TRY(cudaEventRecord(ev_[0].get(), stream_.get()));
        CUDA_TRY(rx::launch_seed_k2pow(buf_, m, t, stream_.get()));
        rc = run_chain(m);
        if (rc != B200POST_OK) return rc;
        uint32_t hit = 0xffffffffu;
        if (difficulty) {
            CUDA_TRY(cudaMemsetAsync(d_found_.get(), 0xff, 4, stream_.get()));
            CUDA_TRY(rx::launch_find_below(buf_, m, d_diff_.get(), d_found_.get(), stream_.get()));
            CUDA_TRY(cudaMemcpyAsync(&hit, d_found_.get(), 4, cudaMemcpyDeviceToHost, stream_.get()));
        }
        if (hashes) CUDA_TRY(cudaMemcpyAsync(h_stage_.get(), buf_.hashes, (size_t)m * 32, cudaMemcpyDeviceToHost, stream_.get()));
        CUDA_TRY(cudaEventRecord(ev_[1].get(), stream_.get()));
        CUDA_TRY(cudaStreamSynchronize(stream_.get()));
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, ev_[0].get(), ev_[1].get()));
        total_ms_ += ms; hashes_ += m;
        if (done) *done += m;
        if (hashes) memcpy(hashes + off * 32, h_stage_.get(), (size_t)m * 32);
        if (difficulty && hit != 0xffffffffu) { if (found) *found = t.start + hit; break; }
    }
    return B200POST_OK;
}

// ------------------------------------------------------------------------------------------------ registry
static std::mutex g_rx_mu;
static std::map<int, std::unique_ptr<RandomxEngine>> &g_rx = *new std::map<int, std::unique_ptr<RandomxEngine>>();

RandomxEngine *randomx_engine_for(uint32_t provider) {
    if (provider == B200POST_CPU_PROVIDER_ID) {
        set_error("provider 0xffffffff (CPU) is not served by libb200post: this library has no CPU path");
        return nullptr;
    }
    const int n = device_count();
    if ((int64_t)provider >= n) { set_error(n == 0 ? "no CUDA device available" : "unknown provider id"); return nullptr; }
    std::lock_guard<std::mutex> lk(g_rx_mu);
    auto it = g_rx.find((int)provider);
    if (it == g_rx.end()) it = g_rx.emplace((int)provider, std::make_unique<RandomxEngine>((int)provider)).first;
    return it->second.get();
}

void randomx_shutdown_all() {
    std::lock_guard<std::mutex> lk(g_rx_mu);
    g_rx.clear();
}

void randomx_release(int device) {
    RandomxEngine *e = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_rx_mu);
        auto it = g_rx.find(device);
        if (it != g_rx.end()) e = it->second.get();
    }
    if (e) e->release();
}

}  // namespace b200post
