// engine.cu — layer scheduler for the POST label kernels (see engine.h).
//
// Mirrors what the reference's initializer does around libpost's `initialize()` (activation/post.go:295:
// batches of ComputeBatchSize labels, cancellable, progress observable) but sized for the GPU.  A *layer*
// is one label per resident slot (threads x SMs that fit the registers and the HBM scratch).  With the
// pipelined ROMix kernel the stream carries, for layer m:
//     K1(m)  ->  K2p{ mix layer m-1 | fill layer m }  ->  K3(m-1)        (and on the copy stream: D2H(m-1))
// so every launch keeps half of each thread's work latency-free, and the 16-byte labels of layer m-1
// leave the device while layer m computes.  Buffers are double-buffered by layer parity; the host thread
// stays one launch ahead of the GPU.
#include "engine.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <vector>

#include "../../include/b200post.h"
#include "metrics.h"

namespace b200post {

Options &options() { static Options o; return o; }
std::atomic<uint64_t> g_launches{0};

static thread_local std::string t_error;
void set_error(const std::string &msg) { t_error = msg; }
const char *last_error() { return t_error.c_str(); }

#define CU_TRY(expr)                                                                                     \
    do {                                                                                                 \
        cudaError_t e__ = (expr);                                                                        \
        if (e__ != cudaSuccess) {                                                                        \
            set_error(std::string(#expr) + ": " + cudaGetErrorString(e__));                              \
            return e__ == cudaErrorMemoryAllocation ? B200POST_ERR_OUT_OF_MEMORY : B200POST_ERR_CUDA;    \
        }                                                                                                \
    } while (0)

static inline uint32_t round_up(uint32_t x, uint32_t m) { return (x + m - 1) / m * m; }

DeviceEngine::DeviceEngine(int device) : dev_(device) { cudaGetDeviceProperties(&prop_, device); }

DeviceEngine::~DeviceEngine() {
    cudaSetDevice(dev_);
    release();
}

void DeviceEngine::release() {
    if (stream_) cudaStreamSynchronize(stream_);
    if (copy_stream_) cudaStreamSynchronize(copy_stream_);
    cudaFree(V_raw_); V_raw_ = nullptr; V_ = nullptr; v_bytes_ = 0; v_align_ = 0;
    for (int b = 0; b < 2; b++) {
        cudaFree(X_[b]); X_[b] = nullptr;
        cudaFree(d_out_[b]); d_out_[b] = nullptr;
        cudaFreeHost(h_out_[b]); h_out_[b] = nullptr;
        cudaFree(d_commit_[b]); d_commit_[b] = nullptr;
        cudaFree(d_idx_[b]); d_idx_[b] = nullptr;
        cudaFreeHost(h_commit_[b]); h_commit_[b] = nullptr;
        cudaFreeHost(h_idx_[b]); h_idx_[b] = nullptr;
        cudaFree(d_cidx_[b]); d_cidx_[b] = nullptr; cudaFreeHost(h_cidx_[b]); h_cidx_[b] = nullptr;
        cudaFree(d_exp_[b]); d_exp_[b] = nullptr; cudaFreeHost(h_exp_[b]); h_exp_[b] = nullptr;
        cudaFree(d_bits_[b]); d_bits_[b] = nullptr;
        cudaFree(d_cnt_[b]); d_cnt_[b] = nullptr; cudaFreeHost(h_cnt_[b]); h_cnt_[b] = nullptr;
        cudaEvent_t *evs[] = {&ev_done_[b], &ev_in_[b], &ev_k3_[b], &ev_k2a_[b], &ev_k2b_[b], &ev_call_[b], &ev_exp_[b]};
        for (cudaEvent_t *e : evs) { if (*e) cudaEventDestroy(*e); *e = nullptr; }
        k2_pending_[b] = false; in_pending_[b] = false; pend_[b].live = false;
    }
    for (int b = 0; b < 2; b++) { if (ev_timer_[b]) cudaEventDestroy(ev_timer_[b]); ev_timer_[b] = nullptr; }
    cudaFree(d_ctab_); d_ctab_ = nullptr; ctab_rows_ = 0;
    cudaFree(d_range_commit_); d_range_commit_ = nullptr;
    cudaFree(d_diff_); d_diff_ = nullptr;
    cudaFree(d_cta_cand_); d_cta_cand_ = nullptr;
    cudaFree(d_running_); d_running_ = nullptr;
    cudaFreeHost(h_running_); h_running_ = nullptr;
    if (stream_) cudaStreamDestroy(stream_);
    if (copy_stream_) cudaStreamDestroy(copy_stream_);
    copy_stream_ = nullptr;
    stream_ = nullptr;
    alloc_slots_ = 0;
    wave_slots_ = 0;
}

// Decide the layer size for scrypt-N and make sure scratch for min(layer, want_slots) slots exists.
int DeviceEngine::ensure(uint64_t N, uint64_t want_slots) {
    Options &o = options();
    const int variant = (int)o.romix_variant.load(), mw = (int)o.rotate_mask.load();
    int tpb = (int)o.tpb.load();
    if (variant != ROMIX_PIPELINED && tpb != 128 && tpb != 256) tpb = 128;   // the classic kernels are built for 128/256 only
    const int dr = (int)o.dr_unroll.load();
    if (!stream_) {
        CU_TRY(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
        CU_TRY(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
        for (int b = 0; b < 2; b++) {
            CU_TRY(cudaEventCreateWithFlags(&ev_done_[b], cudaEventDisableTiming));
            CU_TRY(cudaEventCreateWithFlags(&ev_in_[b], cudaEventDisableTiming));
            CU_TRY(cudaEventCreateWithFlags(&ev_k3_[b], cudaEventDisableTiming));
            CU_TRY(cudaEventCreate(&ev_k2a_[b]));
            CU_TRY(cudaEventCreate(&ev_k2b_[b]));
            CU_TRY(cudaEventCreate(&ev_call_[b]));
            CU_TRY(cudaEventCreateWithFlags(&ev_exp_[b], cudaEventDisableTiming));
            CU_TRY(cudaMalloc(&d_cnt_[b], 4));
            CU_TRY(cudaMallocHost(&h_cnt_[b], 4));
        }
        CU_TRY(cudaMalloc(&d_diff_, 32));
        CU_TRY(cudaMalloc(&d_range_commit_, 32));
        CU_TRY(cudaMalloc(&d_running_, sizeof(VrfCandidate)));
        CU_TRY(cudaMallocHost(&h_running_, sizeof(VrfCandidate)));
    }
    const size_t pads = variant == ROMIX_PIPELINED ? 2 : 1;   // scratchpads per slot
    const size_t per_slot = 128 * (size_t)N * pads;
    size_t free_b = 0, total_b = 0;
    CU_TRY(cudaMemGetInfo(&free_b, &total_b));
    size_t budget = (size_t)((double)(free_b + v_bytes_) * 0.95);   // 0.95: headroom for the k2pow engine's dataset and scratchpads (~14 GiB) when it allocates after this one
    const int64_t cap_mib = o.max_scratch_mib.load();
    if (cap_mib > 0) budget = std::min(budget, (size_t)cap_mib << 20);
    const size_t sms = (size_t)prop_.multiProcessorCount;
    const int64_t want_ctas = o.ctas_per_sm.load();
    // resident CTAs per SM of `t` threads: the occupancy limit, the option, then what the HBM budget holds
    auto ctas_for = [&](int t) {
        int c = romix_max_ctas_per_sm(variant, mw, t, dr);
        if (want_ctas > 0) c = std::min<int>(c, (int)want_ctas);
        while (c > 0 && per_slot * (size_t)t * sms * (size_t)c > budget) c--;
        return c;
    };
    if (romix_max_ctas_per_sm(variant, mw, tpb, dr) <= 0) { set_error("romix kernel cannot be resident (unsupported variant / mask / tpb combination)"); return B200POST_ERR_INVALID_ARGUMENT; }
    int ctas = ctas_for(tpb);
    // HBM, not the register file, bounds the pipelined layer when it cannot give every SM one CTA of `tpb` slots: an
    // 80 GB H100 holds ~36 k slots at N = 8192, while 132 SMs x 512 threads would take 67 k, and a 512-thread grid of
    // 36 k slots leaves half of the SMs idle.  Smaller CTAs (down to 64 threads) then spread the layer over every SM;
    // the size that puts the most slots on the device wins.
    if (variant == ROMIX_PIPELINED) {
        for (int t = tpb / 2; t >= 64; t /= 2) {
            const int c = ctas_for(t);
            if ((uint64_t)c * t > (uint64_t)ctas * tpb) { ctas = c; tpb = t; }
        }
    }
    if (ctas == 0) ctas = 1;   // not even one CTA per SM fits: the layer shrinks below
    variant_ = variant; mw_ = mw; tpb_ = tpb; dr_unroll_ = dr;
    uint64_t wave = (uint64_t)sms * (uint64_t)ctas * (uint64_t)tpb;
    if (per_slot * wave > budget) {
        // not even one CTA per SM: shrink to what fits, in whole warps (the kernels take any multiple of 32)
        wave = budget / per_slot / 32 * 32;
        if (wave == 0) { set_error("not enough HBM for one warp of ROMix scratch"); return B200POST_ERR_OUT_OF_MEMORY; }
    }
    wave_slots_ = (uint32_t)wave;

    const uint32_t need = (uint32_t)std::min<uint64_t>(wave, round_up((uint32_t)std::min<uint64_t>(want_slots, wave), 32));
    const size_t need_v = per_slot * (size_t)need;
    if (need_v > v_bytes_ || 128 * (size_t)N * 32 > v_align_) {
        CU_TRY(cudaStreamSynchronize(stream_));
        cudaFree(V_raw_); V_raw_ = nullptr; V_ = nullptr; v_bytes_ = 0;
        // align to the largest per-warp region this allocation can be used with (N * 4 KiB, <= 4 GiB) so
        // that no region straddles a 4 GiB boundary: the kernels do 32-bit address arithmetic inside one
        const size_t align = std::min<size_t>(128 * (size_t)N * 32, (size_t)1 << 32);
        CU_TRY(cudaMalloc(&V_raw_, need_v + align));
        V_ = reinterpret_cast<uint4 *>(((uintptr_t)V_raw_ + align - 1) / align * align);
        v_bytes_ = need_v;
        v_align_ = align;
    }
    if (need > alloc_slots_) {
        CU_TRY(cudaStreamSynchronize(stream_));
        for (int b = 0; b < 2; b++) {
            cudaFree(X_[b]); cudaFree(d_commit_[b]); cudaFree(d_idx_[b]); cudaFree(d_out_[b]); cudaFree(d_cidx_[b]);
            cudaFreeHost(h_commit_[b]); cudaFreeHost(h_idx_[b]); cudaFreeHost(h_out_[b]); cudaFreeHost(h_cidx_[b]);
            cudaFree(d_exp_[b]); cudaFreeHost(h_exp_[b]); cudaFree(d_bits_[b]);
            d_cidx_[b] = nullptr; h_cidx_[b] = nullptr; d_exp_[b] = nullptr; h_exp_[b] = nullptr; d_bits_[b] = nullptr;
            X_[b] = nullptr; d_commit_[b] = nullptr; d_idx_[b] = nullptr; d_out_[b] = nullptr;
            h_commit_[b] = nullptr; h_idx_[b] = nullptr; h_out_[b] = nullptr;
        }
        cudaFree(d_cta_cand_); d_cta_cand_ = nullptr;
        alloc_slots_ = 0;
        for (int b = 0; b < 2; b++) {
            CU_TRY(cudaMalloc(&X_[b], (size_t)need * 128));
            CU_TRY(cudaMalloc(&d_commit_[b], (size_t)need * 32));
            CU_TRY(cudaMalloc(&d_idx_[b], (size_t)need * 8));
            CU_TRY(cudaMalloc(&d_out_[b], (size_t)need * 16));
            CU_TRY(cudaMallocHost(&h_commit_[b], (size_t)need * 32));
            CU_TRY(cudaMallocHost(&h_idx_[b], (size_t)need * 8));
            CU_TRY(cudaMallocHost(&h_out_[b], (size_t)need * 16));
            CU_TRY(cudaMalloc(&d_cidx_[b], (size_t)need * 4));
            CU_TRY(cudaMallocHost(&h_cidx_[b], (size_t)need * 4));
            CU_TRY(cudaMalloc(&d_exp_[b], (size_t)need * 16));
            CU_TRY(cudaMallocHost(&h_exp_[b], (size_t)need * 16));
            CU_TRY(cudaMalloc(&d_bits_[b], (size_t)need / 32 * 4));
        }
        CU_TRY(cudaMalloc(&d_cta_cand_, (size_t)pbkdf2_final_ctas(need) * sizeof(VrfCandidate)));
        alloc_slots_ = need;
    }
    return B200POST_OK;
}

// collect the ROMix device time recorded under parity `buf` (blocks until that launch has finished)
void DeviceEngine::harvest(int buf) {
    if (!k2_pending_[buf]) return;
    float ms = 0;
    if (cudaEventSynchronize(ev_k2b_[buf]) == cudaSuccess &&
        cudaEventElapsedTime(&ms, ev_k2a_[buf], ev_k2b_[buf]) == cudaSuccess) {
        romix_ms_ += ms; romix_launches_++; romix_labels_ += k2_labels_[buf];
    }
    k2_pending_[buf] = false;
}

int DeviceEngine::retire(const Job &job, int b) {
    if (!pend_[b].live) return B200POST_OK;
    CU_TRY(cudaEventSynchronize(ev_done_[b]));
    if (job.out_host) memcpy(job.out_host + pend_[b].off * 16, h_out_[b], (size_t)pend_[b].n * 16);
    if (job.cmp && *h_cnt_[b]) {
        // rare path: the layer has mismatches; fetch its bitmap and decode positions (ascending: layers retire in order)
        std::vector<uint32_t> bits(round_up(pend_[b].n, 32) / 32);
        CU_TRY(cudaMemcpy(bits.data(), d_bits_[b], bits.size() * 4, cudaMemcpyDeviceToHost));
        job.cmp->mismatches += *h_cnt_[b];
        for (size_t w = 0; w < bits.size() && job.cmp->first.size() < CompareResult::kMaxReported; w++)
            for (uint32_t v = bits[w]; v && job.cmp->first.size() < CompareResult::kMaxReported; v &= v - 1)
                job.cmp->first.push_back(pend_[b].off + 32 * w + (uint64_t)__builtin_ctz(v));
    }
    pend_[b].live = false;
    return B200POST_OK;
}

int DeviceEngine::stage_layer(const Job &job, uint64_t layer, int b, uint32_t n_valid, LabelJob *lj) {
    const uint64_t off = layer * (uint64_t)std::min<uint64_t>(wave_slots_, alloc_slots_);
    if (job.gather && job.commit_index) {
        if (in_pending_[b]) { CU_TRY(cudaEventSynchronize(ev_in_[b])); in_pending_[b] = false; }
        memcpy(h_cidx_[b], job.commit_index + off, (size_t)n_valid * 4);
        memcpy(h_idx_[b], job.indices + off, (size_t)n_valid * 8);
        CU_TRY(cudaMemcpyAsync(d_cidx_[b], h_cidx_[b], (size_t)n_valid * 4, cudaMemcpyHostToDevice, stream_));
        CU_TRY(cudaMemcpyAsync(d_idx_[b], h_idx_[b], (size_t)n_valid * 8, cudaMemcpyHostToDevice, stream_));
        CU_TRY(cudaEventRecord(ev_in_[b], stream_));
        in_pending_[b] = true;
        *lj = LabelJob{reinterpret_cast<const uint32_t *>(d_ctab_), 0, d_idx_[b], 0, n_valid, d_cidx_[b]};
    } else if (job.gather && !job.commitments) {
        // one commitment for every item (compare jobs): only the indices travel
        if (in_pending_[b]) { CU_TRY(cudaEventSynchronize(ev_in_[b])); in_pending_[b] = false; }
        memcpy(h_idx_[b], job.indices + off, (size_t)n_valid * 8);
        CU_TRY(cudaMemcpyAsync(d_idx_[b], h_idx_[b], (size_t)n_valid * 8, cudaMemcpyHostToDevice, stream_));
        CU_TRY(cudaEventRecord(ev_in_[b], stream_));
        in_pending_[b] = true;
        *lj = LabelJob{d_range_commit_, 0, d_idx_[b], 0, n_valid, nullptr};
    } else if (job.gather) {
        if (in_pending_[b]) { CU_TRY(cudaEventSynchronize(ev_in_[b])); in_pending_[b] = false; }
        memcpy(h_commit_[b], job.commitments + off * 32, (size_t)n_valid * 32);
        memcpy(h_idx_[b], job.indices + off, (size_t)n_valid * 8);
        CU_TRY(cudaMemcpyAsync(d_commit_[b], h_commit_[b], (size_t)n_valid * 32, cudaMemcpyHostToDevice, stream_));
        CU_TRY(cudaMemcpyAsync(d_idx_[b], h_idx_[b], (size_t)n_valid * 8, cudaMemcpyHostToDevice, stream_));
        CU_TRY(cudaEventRecord(ev_in_[b], stream_));
        in_pending_[b] = true;
        *lj = LabelJob{reinterpret_cast<const uint32_t *>(d_commit_[b]), 8, d_idx_[b], 0, n_valid, nullptr};
    } else {
        *lj = LabelJob{d_range_commit_, 0, nullptr, job.start + off, n_valid, nullptr};
    }
    CU_TRY(launch_pbkdf2_expand(*lj, X_[b], alloc_slots_, round_up(n_valid, 32), stream_));
    g_launches += 1;
    return B200POST_OK;
}

int DeviceEngine::finish_layer(const Job &job, uint64_t layer, int b, uint32_t n_valid, const LabelJob &lj) {
    const uint64_t off = layer * (uint64_t)std::min<uint64_t>(wave_slots_, alloc_slots_);
    const uint32_t n_slots = round_up(n_valid, 32);
    if (job.expect_host) {
        // K3c: the expected slice goes H2D on the copy stream (pinned staging, double-buffered by parity; retire(b) has
        // seen the previous copy out of h_exp_[b] finish), and K3c waits for it by event
        memcpy(h_exp_[b], job.expect_host + off * 16, (size_t)n_valid * 16);
        CU_TRY(cudaMemcpyAsync(d_exp_[b], h_exp_[b], (size_t)n_valid * 16, cudaMemcpyHostToDevice, copy_stream_));
        CU_TRY(cudaEventRecord(ev_exp_[b], copy_stream_));
        CU_TRY(cudaStreamWaitEvent(stream_, ev_exp_[b], 0));
        CU_TRY(cudaMemsetAsync(d_cnt_[b], 0, 4, stream_));
        CU_TRY(launch_pbkdf2_final_compare(lj, X_[b], alloc_slots_, n_slots, d_exp_[b], d_bits_[b], d_cnt_[b], job.d_diff,
                                           d_cta_cand_, stream_));
    } else {
        uint8_t *d_out = job.out_dev ? job.out_dev + off * 16 : d_out_[b];
        CU_TRY(launch_pbkdf2_final(lj, X_[b], alloc_slots_, n_slots, d_out, job.d_diff, d_cta_cand_, stream_));
    }
    g_launches += 1;
    if (job.d_diff) {
        CU_TRY(launch_vrf_merge(d_cta_cand_, pbkdf2_final_ctas(n_slots), d_running_, stream_));
        g_launches += 1;
    }
    if (job.out_host) {
        // the copy runs on its own stream: the next layers' kernels do not queue behind PCIe
        CU_TRY(cudaEventRecord(ev_k3_[b], stream_));
        CU_TRY(cudaStreamWaitEvent(copy_stream_, ev_k3_[b], 0));
        CU_TRY(cudaMemcpyAsync(h_out_[b], d_out_[b], (size_t)n_valid * 16, cudaMemcpyDeviceToHost, copy_stream_));
        CU_TRY(cudaEventRecord(ev_done_[b], copy_stream_));
    } else if (job.expect_host) {
        // only the 4-byte count comes back per layer; the bitmap follows in retire() when it is non-zero
        CU_TRY(cudaEventRecord(ev_k3_[b], stream_));
        CU_TRY(cudaStreamWaitEvent(copy_stream_, ev_k3_[b], 0));
        CU_TRY(cudaMemcpyAsync(h_cnt_[b], d_cnt_[b], 4, cudaMemcpyDeviceToHost, copy_stream_));
        CU_TRY(cudaEventRecord(ev_done_[b], copy_stream_));
    } else {
        CU_TRY(cudaEventRecord(ev_done_[b], stream_));
    }
    pend_[b] = Pending{off, n_valid, true};
    return B200POST_OK;
}

int DeviceEngine::run_job(const Job &job) {
    const uint64_t S = std::min<uint64_t>(wave_slots_, alloc_slots_);
    const uint64_t M = (job.total + S - 1) / S;
    int rc_ = B200POST_OK, status = B200POST_OK;
    auto layer_count = [&](uint64_t m) { return (uint32_t)std::min<uint64_t>(S, job.total - m * S); };

    // small jobs (a proof's K2 labels, one VRF-nonce label, ...): the low-latency kernel, one launch
    const int64_t lowlat_max = options().lowlat_max_labels.load();
    const bool lowlat = variant_ == ROMIX_PIPELINED && M == 1 && lowlat_max > 0 && job.total <= (uint64_t)lowlat_max &&
                        job.total <= (uint64_t)prop_.multiProcessorCount * 4 * 32;
    if (lowlat) {
        spec_.valid = false;
        if (job.cancel && *job.cancel) return B200POST_ERR_CANCELLED;
        for (int b = 0; b < 2; b++) { if ((rc_ = retire(job, b))) return rc_; harvest(b); }
        const uint32_t n_valid = (uint32_t)job.total;
        LabelJob lj;
        if ((rc_ = stage_layer(job, 0, 0, n_valid, &lj))) return rc_;
        RomixParams rp;
        rp.V = V_; rp.X = X_[0]; rp.x_stride = alloc_slots_; rp.N = (uint32_t)job.N; rp.n_slots = n_valid; rp.flags = 0;
        CU_TRY(cudaEventRecord(ev_k2a_[0], stream_));
        CU_TRY(launch_romix_lowlat(mw_, rp, romix_lowlat_warps(n_valid, prop_.multiProcessorCount), stream_));
        CU_TRY(cudaEventRecord(ev_k2b_[0], stream_));
        k2_pending_[0] = true; k2_labels_[0] = n_valid;
        g_launches += 1;
        if ((rc_ = finish_layer(job, 0, 0, n_valid, lj))) return rc_;
    } else if (variant_ != ROMIX_PIPELINED) {
        spec_.valid = false;
        for (uint64_t m = 0; m < M; m++) {
            if (job.cancel && *job.cancel) { status = B200POST_ERR_CANCELLED; break; }
            const int b = (int)(m & 1);
            if ((rc_ = retire(job, b))) return rc_;
            harvest(b);
            const uint32_t n_valid = layer_count(m);
            LabelJob lj;
            if ((rc_ = stage_layer(job, m, b, n_valid, &lj))) return rc_;
            RomixParams rp;
            rp.V = V_; rp.X = X_[b]; rp.x_stride = alloc_slots_; rp.N = (uint32_t)job.N; rp.n_slots = round_up(n_valid, 32);
            rp.flags = (uint32_t)options().debug_skip_phase.load();
            CU_TRY(cudaEventRecord(ev_k2a_[b], stream_));
            CU_TRY(launch_romix(variant_, mw_, tpb_, rp, stream_));
            CU_TRY(cudaEventRecord(ev_k2b_[b], stream_));
            k2_pending_[b] = true; k2_labels_[b] = n_valid;
            g_launches += 1;
            if ((rc_ = finish_layer(job, m, b, n_valid, lj))) return rc_;
        }
    } else {
        // consume a matching speculation: layer 0 of this call was filled by the previous call's last launch
        const bool resume = !job.gather && spec_.valid && spec_.N == job.N && spec_.next_start == job.start && spec_.slots == S &&
                            spec_.alloc_slots == alloc_slots_ && spec_.V == V_ && !memcmp(spec_.commitment, cur_commitment_, 32);
        const int poff = resume ? spec_.parity : 0;
        spec_.valid = false;
        const bool speculate = !job.gather && options().speculate_next.load() != 0 && M >= 4 && job.start + job.total + S > job.start + job.total;
        auto par = [&](uint64_t m) { return (int)((m + (uint64_t)poff) & 1); };
        LabelJob lj[2];
        uint32_t nv[2] = {0, 0};
        bool spec_filled = false;
        for (uint64_t m = 0; m <= M; m++) {
            if (m < M && job.cancel && *job.cancel) { status = B200POST_ERR_CANCELLED; break; }
            const int b = par(m);
            harvest(b);
            bool fill = false;
            uint32_t n_fill = 0;
            if (m < M) {
                nv[b] = layer_count(m);
                if (m == 0 && resume) {
                    lj[b] = LabelJob{d_range_commit_, 0, nullptr, job.start, nv[b], nullptr};   // already filled: X_[b] holds its mid-state
                } else {
                    if ((rc_ = stage_layer(job, m, b, nv[b], &lj[b]))) return rc_;
                    fill = true; n_fill = round_up(nv[b], 32);
                }
            } else if (speculate && status == B200POST_OK) {
                // one layer past the end of this call: the next initialize() batch, if it comes
                LabelJob next;
                Job after = job;                       // the range that would follow this call: [start + total, ...)
                after.start = job.start + job.total;
                if ((rc_ = stage_layer(after, 0, b, (uint32_t)S, &next))) return rc_;
                fill = true; n_fill = (uint32_t)S; spec_filled = true;
            }
            const uint32_t n_mix = m >= 1 ? round_up(nv[b ^ 1], 32) : 0;
            if (n_fill == 0 && n_mix == 0) continue;   // resumed call: nothing to launch for m = 0
            PipeParams pp;
            pp.V = V_; pp.x_stride = alloc_slots_; pp.N = (uint32_t)job.N;
            pp.Xfill = X_[b]; pp.Xmix = X_[b ^ 1];
            pp.n_fill = n_fill;
            pp.n_mix = n_mix;
            pp.fill_parity = (uint32_t)b;
            pp.cta_trace = nullptr;
            // diagnostics: B200POST_CTA_TRACE=<file> dumps {start ns, end ns, smid} per CTA of the last steady launch
            static const char *trace_path = getenv("B200POST_CTA_TRACE");
            unsigned long long *d_trace = nullptr;
            const uint32_t n_cta = (std::max(pp.n_fill, pp.n_mix) + tpb_ - 1) / tpb_;
            if (trace_path && m >= 1 && m + 1 == M) {
                CU_TRY(cudaMalloc(&d_trace, (size_t)n_cta * 24));
                CU_TRY(cudaMemsetAsync(d_trace, 0, (size_t)n_cta * 24, stream_));
                pp.cta_trace = d_trace;
            }
            CU_TRY(cudaEventRecord(ev_k2a_[b], stream_));
            CU_TRY(launch_romix_pipe(mw_, tpb_, dr_unroll_, pp, stream_));
            CU_TRY(cudaEventRecord(ev_k2b_[b], stream_));
            k2_pending_[b] = true;
            k2_labels_[b] = 0.5 * ((fill ? (m < M ? nv[b] : (uint32_t)S) : 0) + (m >= 1 ? nv[b ^ 1] : 0));
            g_launches += 1;
            if (d_trace) {
                std::vector<unsigned long long> h((size_t)n_cta * 3);
                CU_TRY(cudaMemcpyAsync(h.data(), d_trace, h.size() * 8, cudaMemcpyDeviceToHost, stream_));
                CU_TRY(cudaStreamSynchronize(stream_));
                cudaFree(d_trace);
                if (FILE *f = fopen(trace_path, "w")) {
                    for (uint32_t c = 0; c < n_cta; c++) fprintf(f, "%u,%llu,%llu,%llu\n", c, h[3 * c], h[3 * c + 1], h[3 * c + 2]);
                    fclose(f);
                }
            }
            if (m >= 1) {
                // layer m-3 used the output buffers of this parity.  Waiting for it HERE, after launch m is queued,
                // keeps one whole launch ahead of the host: a slow wake-up, host copy or PCIe transfer does not
                // leave the GPU idle between layers.
                if ((rc_ = retire(job, b ^ 1))) return rc_;
                if ((rc_ = finish_layer(job, m - 1, b ^ 1, nv[b ^ 1], lj[b ^ 1]))) return rc_;
            }
        }
        if (spec_filled && status == B200POST_OK) {
            spec_.valid = true; spec_.N = job.N; spec_.next_start = job.start + job.total; spec_.parity = par(M);
            spec_.slots = (uint32_t)S; spec_.alloc_slots = alloc_slots_; spec_.V = V_;
            memcpy(spec_.commitment, cur_commitment_, 32);
        }
    }
    for (int b = 0; b < 2; b++) {
        if ((rc_ = retire(job, b))) return rc_;
        harvest(b);
        if (in_pending_[b]) { CU_TRY(cudaEventSynchronize(ev_in_[b])); in_pending_[b] = false; }
    }
    return status;
}

int DeviceEngine::labels_range(const uint8_t commitment[32], uint64_t N, uint64_t start, uint64_t count, uint8_t *out_host,
                               uint8_t *out_dev, const uint8_t *vrf_difficulty, VrfResult *vrf, const volatile int *cancel) {
    return range_call(commitment, N, start, count, out_host, out_dev, nullptr, nullptr, vrf_difficulty, vrf, cancel);
}

int DeviceEngine::labels_compare_range(const uint8_t commitment[32], uint64_t N, uint64_t start, uint64_t count,
                                       const uint8_t *expect_host, const uint8_t *vrf_difficulty, VrfResult *vrf,
                                       CompareResult *cmp, const volatile int *cancel) {
    if (!expect_host || !cmp) { set_error("compare job without expected labels or result"); return B200POST_ERR_INVALID_ARGUMENT; }
    return range_call(commitment, N, start, count, nullptr, nullptr, expect_host, cmp, vrf_difficulty, vrf, cancel);
}

int DeviceEngine::range_call(const uint8_t commitment[32], uint64_t N, uint64_t start, uint64_t count, uint8_t *out_host,
                             uint8_t *out_dev, const uint8_t *expect_host, CompareResult *cmp, const uint8_t *vrf_difficulty,
                             VrfResult *vrf, const volatile int *cancel) {
    std::lock_guard<std::mutex> lk(mu_);
    CU_TRY(cudaSetDevice(dev_));
    if (vrf) *vrf = VrfResult{};
    if (cmp) *cmp = CompareResult{};
    if (count == 0) return B200POST_OK;
    int rc = ensure(N, count);
    if (rc) return rc;
    CU_TRY(cudaEventRecord(ev_call_[0], stream_));

    // per-call constants: commitment, VRF threshold, running candidate
    memcpy(cur_commitment_, commitment, 32);
    CU_TRY(cudaMemcpyAsync(d_range_commit_, commitment, 32, cudaMemcpyHostToDevice, stream_));
    Job job;
    job.start = start; job.total = count; job.N = N; job.out_host = out_host; job.out_dev = out_dev; job.cancel = cancel;
    job.expect_host = expect_host; job.cmp = cmp;
    if (vrf_difficulty) {
        uint32_t be[8];
        for (int k = 0; k < 8; k++)
            be[k] = ((uint32_t)vrf_difficulty[4 * k] << 24) | ((uint32_t)vrf_difficulty[4 * k + 1] << 16) |
                    ((uint32_t)vrf_difficulty[4 * k + 2] << 8) | vrf_difficulty[4 * k + 3];
        CU_TRY(cudaMemcpyAsync(d_diff_, be, 32, cudaMemcpyHostToDevice, stream_));
        CU_TRY(cudaMemsetAsync(d_running_, 0, sizeof(VrfCandidate), stream_));
        CU_TRY(cudaStreamSynchronize(stream_));   // `be` is a stack buffer
        job.d_diff = d_diff_;
    }
    const int status = run_job(job);
    if (status != B200POST_OK && status != B200POST_ERR_CANCELLED) { quiesce(); return status; }
    if (status == B200POST_OK && vrf_difficulty && vrf) {
        CU_TRY(cudaMemcpyAsync(h_running_, d_running_, sizeof(VrfCandidate), cudaMemcpyDeviceToHost, stream_));
        CU_TRY(cudaStreamSynchronize(stream_));
        vrf->found = h_running_->found != 0;
        if (vrf->found) {
            vrf->index = h_running_->index;
            for (int k = 0; k < 8; k++) {
                const uint32_t v = h_running_->label_be[k];
                vrf->label32[4 * k] = (uint8_t)(v >> 24); vrf->label32[4 * k + 1] = (uint8_t)(v >> 16);
                vrf->label32[4 * k + 2] = (uint8_t)(v >> 8); vrf->label32[4 * k + 3] = (uint8_t)v;
            }
        }
    }
    CU_TRY(cudaEventRecord(ev_call_[1], stream_));
    CU_TRY(cudaStreamSynchronize(stream_));
    { float ms = 0; if (cudaEventElapsedTime(&ms, ev_call_[0], ev_call_[1]) == cudaSuccess) last_call_ms_ = ms; }
    metrics().range_calls_total++; metrics().device_ns_total += (uint64_t)(last_call_ms_ * 1e6);
    if (status == B200POST_OK && !expect_host) metrics().labels_range_total += count;
    if (status == B200POST_ERR_CANCELLED) set_error("cancelled");
    return status;
}

int DeviceEngine::labels_gather(size_t n_items, const uint8_t *commitments, const uint64_t *indices, uint64_t N, uint8_t *out_host,
                                uint8_t *out_dev) {
    std::lock_guard<std::mutex> lk(mu_);
    CU_TRY(cudaSetDevice(dev_));
    if (n_items == 0) return B200POST_OK;
    int rc = ensure(N, n_items);
    if (rc) return rc;
    CU_TRY(cudaEventRecord(ev_call_[0], stream_));
    Job job;
    spec_.valid = false;   // the scratch is about to be reused
    job.gather = true; job.commitments = commitments; job.indices = indices; job.total = n_items; job.N = N;
    job.out_host = out_host; job.out_dev = out_dev;
    if ((rc = run_job(job))) { quiesce(); return rc; }
    CU_TRY(cudaEventRecord(ev_call_[1], stream_));
    CU_TRY(cudaStreamSynchronize(stream_));
    { float ms = 0; if (cudaEventElapsedTime(&ms, ev_call_[0], ev_call_[1]) == cudaSuccess) last_call_ms_ = ms; }
    metrics().gather_calls_total++; metrics().labels_gather_total += n_items; metrics().device_ns_total += (uint64_t)(last_call_ms_ * 1e6);
    return B200POST_OK;
}

// After a failed job: drain the stream and forget every in-flight buffer, so that the next call starts clean
// (the error text of the failure is preserved).
void DeviceEngine::quiesce() {
    const std::string keep = last_error();
    if (stream_) cudaStreamSynchronize(stream_);
    if (copy_stream_) cudaStreamSynchronize(copy_stream_);
    cudaGetLastError();
    for (int b = 0; b < 2; b++) { pend_[b].live = false; k2_pending_[b] = false; in_pending_[b] = false; }
    spec_.valid = false;
    set_error(keep);
}

int DeviceEngine::labels_gather_indexed(size_t n_items, size_t n_commit, const uint8_t *commitments, const uint32_t *commit_index,
                                        const uint64_t *indices, uint64_t N, uint8_t *out_host, uint8_t *out_dev) {
    std::lock_guard<std::mutex> lk(mu_);
    CU_TRY(cudaSetDevice(dev_));
    if (n_items == 0) return B200POST_OK;
    int rc = ensure(N, n_items);
    if (rc) return rc;
    if (n_commit > ctab_rows_) {
        CU_TRY(cudaStreamSynchronize(stream_));
        cudaFree(d_ctab_); d_ctab_ = nullptr; ctab_rows_ = 0;
        CU_TRY(cudaMalloc(&d_ctab_, n_commit * 32));
        ctab_rows_ = n_commit;
    }
    CU_TRY(cudaEventRecord(ev_call_[0], stream_));
    CU_TRY(cudaMemcpyAsync(d_ctab_, commitments, n_commit * 32, cudaMemcpyHostToDevice, stream_));
    spec_.valid = false;   // the scratch is about to be reused
    Job job;
    job.gather = true; job.commit_index = commit_index; job.indices = indices; job.total = n_items; job.N = N;
    job.out_host = out_host; job.out_dev = out_dev;
    if ((rc = run_job(job))) { quiesce(); return rc; }
    CU_TRY(cudaEventRecord(ev_call_[1], stream_));
    CU_TRY(cudaStreamSynchronize(stream_));
    { float ms = 0; if (cudaEventElapsedTime(&ms, ev_call_[0], ev_call_[1]) == cudaSuccess) last_call_ms_ = ms; }
    metrics().gather_calls_total++; metrics().labels_gather_total += n_items; metrics().device_ns_total += (uint64_t)(last_call_ms_ * 1e6);
    return B200POST_OK;
}

int DeviceEngine::labels_compare_indexed(const uint8_t commitment[32], size_t n_items, const uint64_t *indices, uint64_t N,
                                         const uint8_t *expect_host, CompareResult *cmp, const volatile int *cancel) {
    std::lock_guard<std::mutex> lk(mu_);
    CU_TRY(cudaSetDevice(dev_));
    if (!commitment || !indices || !expect_host || !cmp) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    *cmp = CompareResult{};
    if (n_items == 0) return B200POST_OK;
    int rc = ensure(N, n_items);
    if (rc) return rc;
    CU_TRY(cudaEventRecord(ev_call_[0], stream_));
    spec_.valid = false;   // the scratch is about to be reused
    memcpy(cur_commitment_, commitment, 32);
    CU_TRY(cudaMemcpyAsync(d_range_commit_, commitment, 32, cudaMemcpyHostToDevice, stream_));
    CU_TRY(cudaStreamSynchronize(stream_));   // `commitment` belongs to the caller
    Job job;
    job.gather = true; job.indices = indices; job.total = n_items; job.N = N;
    job.expect_host = expect_host; job.cmp = cmp; job.cancel = cancel;
    if ((rc = run_job(job))) {
        quiesce();
        if (rc == B200POST_ERR_CANCELLED) set_error("cancelled");
        return rc;
    }
    CU_TRY(cudaEventRecord(ev_call_[1], stream_));
    CU_TRY(cudaStreamSynchronize(stream_));
    { float ms = 0; if (cudaEventElapsedTime(&ms, ev_call_[0], ev_call_[1]) == cudaSuccess) last_call_ms_ = ms; }
    metrics().gather_calls_total++; metrics().device_ns_total += (uint64_t)(last_call_ms_ * 1e6);
    return B200POST_OK;
}

uint32_t DeviceEngine::wave_slots(uint64_t N) {
    std::lock_guard<std::mutex> lk(mu_);
    if (cudaSetDevice(dev_) != cudaSuccess) return 0;
    if (ensure(N, 32) != B200POST_OK) return 0;
    return wave_slots_;
}

int DeviceEngine::timer_mark(int which) {
    std::lock_guard<std::mutex> lk(mu_);
    CU_TRY(cudaSetDevice(dev_));
    if (which < 0 || which > 1) return B200POST_ERR_INVALID_ARGUMENT;
    if (!stream_) { int rc = ensure(2, 32); if (rc) return rc; }
    if (!ev_timer_[which]) CU_TRY(cudaEventCreate(&ev_timer_[which]));
    CU_TRY(cudaEventRecord(ev_timer_[which], stream_));
    return B200POST_OK;
}

double DeviceEngine::timer_elapsed_ms() {
    std::lock_guard<std::mutex> lk(mu_);
    if (!ev_timer_[0] || !ev_timer_[1] || cudaSetDevice(dev_) != cudaSuccess) return -1.0;
    float ms = 0;
    if (cudaEventSynchronize(ev_timer_[1]) != cudaSuccess || cudaEventElapsedTime(&ms, ev_timer_[0], ev_timer_[1]) != cudaSuccess) return -1.0;
    return ms;
}

double DeviceEngine::last_call_ms() {
    std::lock_guard<std::mutex> lk(mu_);
    return last_call_ms_;
}

void DeviceEngine::romix_time(double *ms_total, uint64_t *launches, double *labels, bool reset) {
    std::lock_guard<std::mutex> lk(mu_);
    if (ms_total) *ms_total = romix_ms_;
    if (launches) *launches = romix_launches_;
    if (labels) *labels = romix_labels_;
    if (reset) { romix_ms_ = 0; romix_launches_ = 0; romix_labels_ = 0; }
}

// ------------------------------------------------------------------------------------------------ registry
static std::mutex g_reg_mu;
// heap-allocated and never destroyed at exit: static destructors may run after the CUDA runtime has
// torn down, where cudaFree is no longer legal.  b200post_shutdown() releases explicitly.
static std::map<int, std::unique_ptr<DeviceEngine>> &g_engines = *new std::map<int, std::unique_ptr<DeviceEngine>>();

int device_count() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

DeviceEngine *engine_for(uint32_t provider) {
    if (provider == B200POST_CPU_PROVIDER_ID) {
        set_error("provider 0xffffffff (CPU) is not served by libb200post: this library has no CPU path");
        return nullptr;
    }
    const int n = device_count();
    if ((int64_t)provider >= n) {
        set_error(n == 0 ? "no CUDA device available" : "unknown provider id");
        return nullptr;
    }
    std::lock_guard<std::mutex> lk(g_reg_mu);
    auto it = g_engines.find((int)provider);
    if (it == g_engines.end()) it = g_engines.emplace((int)provider, std::make_unique<DeviceEngine>((int)provider)).first;
    return it->second.get();
}

void shutdown_all() {
    std::lock_guard<std::mutex> lk(g_reg_mu);
    g_engines.clear();
}

}  // namespace b200post
