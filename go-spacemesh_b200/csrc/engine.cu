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
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <thread>
#include <vector>

#include "../../include/b200post.h"
#include "../../include/b200post_setup.h"
#include "metrics.h"

namespace b200post {

Options &options() { static Options o; return o; }
std::atomic<uint64_t> g_launches{0};

static thread_local std::string t_error;
void set_error(const std::string &msg) { t_error = msg; }
const char *last_error() { return t_error.c_str(); }
int fail(int rc, const std::string &msg) { set_error(msg); return rc; }

static inline uint32_t round_up(uint32_t x, uint32_t m) { return (x + m - 1) / m * m; }

DeviceEngine::DeviceEngine(int device) : dev_(device) { cudaGetDeviceProperties(&prop_, device); }

DeviceEngine::~DeviceEngine() {
    // the members free themselves after this body, on this device and with no work of the engine in flight
    cudaSetDevice(dev_);
    if (stream_.get()) cudaStreamSynchronize(stream_.get());
    if (copy_stream_.get()) cudaStreamSynchronize(copy_stream_.get());
}

int DeviceEngine::Layer::allocate(uint32_t slots) {
    CUDA_TRY(X.resize((size_t)slots * 8));
    CUDA_TRY(d_out.resize((size_t)slots * 16));
    CUDA_TRY(h_out.resize((size_t)slots * 16));
    CUDA_TRY(d_commit.resize((size_t)slots * 32));
    CUDA_TRY(h_commit.resize((size_t)slots * 32));
    CUDA_TRY(d_idx.resize(slots));
    CUDA_TRY(h_idx.resize(slots));
    CUDA_TRY(d_cidx.resize(slots));
    CUDA_TRY(h_cidx.resize(slots));
    CUDA_TRY(d_exp.resize((size_t)slots * 16));
    CUDA_TRY(h_exp.resize((size_t)slots * 16));
    CUDA_TRY(d_bits.resize(slots / 32));
    CUDA_TRY(d_cnt.resize(slots / 32));   // a compare job's count in word 0; rider compare chunks' at slot / 32
    CUDA_TRY(h_cnt.resize(slots / 32));
    CUDA_TRY(ev_done.create(cudaEventDisableTiming));
    CUDA_TRY(ev_k3.create(cudaEventDisableTiming));
    CUDA_TRY(ev_in.create(cudaEventDisableTiming));
    CUDA_TRY(ev_exp.create(cudaEventDisableTiming));
    CUDA_TRY(ev_k2a.create(cudaEventDefault));
    CUDA_TRY(ev_k2b.create(cudaEventDefault));
    in_pending = k2_pending = false;
    pend.live = false;
    pend.riders.clear();
    return B200POST_OK;
}

// Decide the layer size for scrypt-N and make sure scratch for min(layer, want_slots) slots exists.
int DeviceEngine::ensure(uint64_t N, uint64_t want_slots) {
    Options &o = options();
    const int variant = (int)o.romix_variant.load(), mw = (int)o.rotate_mask.load();
    int tpb = (int)o.tpb.load();
    const bool two_pads = variant == ROMIX_PIPELINED || variant == ROMIX_PHASED;   // two scratchpads per slot
    if (!two_pads && tpb != 128 && tpb != 256) tpb = 128;   // the classic kernels are built for 128/256 only
    const int dr = (int)o.dr_unroll.load();
    if (!stream_.get()) {
        CUDA_TRY(stream_.create(cudaStreamNonBlocking));
        CUDA_TRY(copy_stream_.create(cudaStreamNonBlocking));
        for (Event &e : ev_call_) CUDA_TRY(e.create(cudaEventDefault));
        CUDA_TRY(d_diff_.resize(8));
        CUDA_TRY(d_range_commit_.resize(8));
        CUDA_TRY(d_running_.resize(1));
        CUDA_TRY(h_running_.resize(1));
    }
    const size_t pads = two_pads ? 2 : 1;   // scratchpads per slot
    const size_t per_slot = 128 * (size_t)N * pads;
    size_t free_b = 0, total_b = 0;
    CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
    // V is aligned to the largest per-warp region it can be used with (N * 4 KiB, <= 4 GiB), so that no region straddles
    // a 4 GiB boundary: the kernels do 32-bit address arithmetic inside one.  The allocation carries that alignment as a
    // pad, which the budget pays for: 95 % of the HBM that is free or held by V (its pad included), less the pad of a V
    // for this N.  So the layer does not depend on what V held before, and V plus its pad fits in the share.
    const size_t align = std::min<size_t>(128 * (size_t)N * 32, (size_t)1 << 32);
    const size_t held = V_ ? v_bytes_ + v_align_ : 0;
    const size_t share = (size_t)((double)(free_b + held) * 0.95);   // 0.95: headroom for the k2pow engine's dataset and scratchpads (~14 GiB) when it allocates after this one
    size_t budget = share > align ? share - align : 0;
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
    if (two_pads) {
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
    if (wave != wave_slots_) spec_.valid = false;   // a pre-filled layer has the old layer's shape
    wave_slots_ = (uint32_t)wave;
    // a phased layer gives each slot two labels of the layer (its two scratchpads)
    const uint64_t layer = variant == ROMIX_PHASED ? 2 * wave : wave;
    layer_labels_ = (uint32_t)layer;

    const uint32_t need = (uint32_t)std::min<uint64_t>(layer, round_up((uint32_t)std::min<uint64_t>(want_slots, layer), 32));
    const size_t need_v = per_slot * (size_t)std::min<uint64_t>(need, wave);
    if (need_v > v_bytes_ || 128 * (size_t)N * 32 > v_align_) {
        CUDA_TRY(cudaStreamSynchronize(stream_.get()));
        spec_.valid = false;
        V_raw_.reset(); V_ = nullptr; v_bytes_ = 0;
        CUDA_TRY(V_raw_.resize(need_v + align));
        V_ = reinterpret_cast<uint4 *>(((uintptr_t)V_raw_.get() + align - 1) / align * align);
        v_bytes_ = need_v;
        v_align_ = align;
    }
    if (need > alloc_slots_) {
        CUDA_TRY(cudaStreamSynchronize(stream_.get()));
        spec_.valid = false;
        alloc_slots_ = 0;
        for (Layer &l : layer_) { int rc = l.allocate(need); if (rc) return rc; }
        CUDA_TRY(d_cta_cand_.resize(pbkdf2_final_ctas(need)));
        alloc_slots_ = need;
    }
    return B200POST_OK;
}

// collect the ROMix device time recorded under parity `buf` (blocks until that launch has finished)
void DeviceEngine::harvest(int buf) {
    Layer &l = layer_[buf];
    if (!l.k2_pending) return;
    float ms = 0;
    if (cudaEventSynchronize(l.ev_k2b.get()) == cudaSuccess &&
        cudaEventElapsedTime(&ms, l.ev_k2a.get(), l.ev_k2b.get()) == cudaSuccess) {
        romix_ms_ += ms; romix_launches_++; romix_labels_ += l.k2_labels;
    }
    l.k2_pending = false;
}

int DeviceEngine::retire(const Job &job, int b) {
    Layer &l = layer_[b];
    if (!l.pend.live) return B200POST_OK;
    CUDA_TRY(cudaEventSynchronize(l.ev_done.get()));
    const LayerPlan &p = l.pend.plan;
    if (job.out_host) memcpy(job.out_host + p.range_off * 16, l.h_out.get(), (size_t)p.n_range * 16);
    // compare results: the layer's (or a rider chunk's) mismatch count, then, only when it is non-zero, its bitmap,
    // decoded into positions of `cmp`'s job from item `first` on (ascending: layers retire in order)
    auto take_mismatches = [&](CompareResult *cmp, uint32_t count, uint32_t word0, uint32_t n, uint64_t first) -> int {
        if (!count) return B200POST_OK;
        std::vector<uint32_t> bits(round_up(n, 32) / 32);
        CUDA_TRY(cudaMemcpy(bits.data(), l.d_bits.get() + word0, bits.size() * 4, cudaMemcpyDeviceToHost));
        cmp->mismatches += count;
        for (size_t w = 0; w < bits.size() && cmp->first.size() < CompareResult::kMaxReported; w++)
            for (uint32_t v = bits[w]; v && cmp->first.size() < CompareResult::kMaxReported; v &= v - 1)
                cmp->first.push_back(first + 32 * w + (uint64_t)__builtin_ctz(v));
        return B200POST_OK;
    };
    if (job.cmp)
        if (int rc = take_mismatches(job.cmp, *l.h_cnt.get(), 0, p.n_range, p.range_off)) return rc;
    for (size_t k = 0; k < p.chunks.size(); k++) {
        const RiderChunk &c = p.chunks[k];
        const Job &rj = *l.pend.riders[k]->job;
        if (rj.out_host) memcpy(rj.out_host + c.item_off * 16, l.h_out.get() + (size_t)c.slot * 16, (size_t)c.n * 16);
        if (rj.cmp)
            if (int rc = take_mismatches(rj.cmp, l.h_cnt.get()[c.slot / 32], c.slot / 32, c.n, c.item_off)) return rc;
    }
    l.pend.live = false;
    if (!p.chunks.empty()) {
        // a rider whose every item has retired is done: it leaves the queue, and its caller returns
        std::lock_guard<std::mutex> lk(rider_mu_);
        for (size_t k = 0; k < p.chunks.size(); k++) {
            Rider *r = l.pend.riders[k];
            r->retired += p.chunks[k].n;
            if (r->retired == r->load.items) {
                r->done = true;
                riders_.erase(std::find(riders_.begin(), riders_.end(), r));
            }
        }
        rider_cv_.notify_all();
    }
    l.pend.riders.clear();
    return B200POST_OK;
}

void DeviceEngine::next_layer(const Job &job, uint64_t range_off, uint64_t S, bool host, Layer &l) {
    l.chunk_rider.clear();
    if (!host) { l.plan = plan_layer((uint32_t)S, range_off, job.total, {}); return; }
    std::lock_guard<std::mutex> lk(rider_mu_);
    std::vector<RiderLoad *> queue;
    for (Rider *r : riders_) queue.push_back(&r->load);
    l.plan = plan_layer((uint32_t)S, range_off, job.total, queue);
    for (const RiderChunk &c : l.plan.chunks) l.chunk_rider.push_back(riders_[c.rider]);
}

int DeviceEngine::stage_layer(const Job &job, int b, LabelJob *lj) {
    Layer &l = layer_[b];
    const LayerPlan &p = l.plan;
    const uint64_t off = p.range_off;
    const uint32_t n_valid = p.n_range;
    *lj = LabelJob{d_range_commit_.get(), 0, nullptr, job.start + off, n_valid, nullptr};
    const bool riders = !p.chunks.empty();
    // the staging buffers of this parity are free once the previous layer's inputs have left them
    if ((job.gather || riders) && l.in_pending) { CUDA_TRY(cudaEventSynchronize(l.ev_in.get())); l.in_pending = false; }
    if (job.gather) {
        memcpy(l.h_idx.get(), job.indices + off, (size_t)n_valid * 8);
        CUDA_TRY(cudaMemcpyAsync(l.d_idx.get(), l.h_idx.get(), (size_t)n_valid * 8, cudaMemcpyHostToDevice, stream_.get()));
        lj->indices = l.d_idx.get();
        lj->start = 0;
        if (job.commit_index) {
            memcpy(l.h_cidx.get(), job.commit_index + off, (size_t)n_valid * 4);
            CUDA_TRY(cudaMemcpyAsync(l.d_cidx.get(), l.h_cidx.get(), (size_t)n_valid * 4, cudaMemcpyHostToDevice, stream_.get()));
            lj->commit = reinterpret_cast<const uint32_t *>(d_ctab_.get());
            lj->commit_index = l.d_cidx.get();
        } else if (job.commitments) {
            memcpy(l.h_commit.get(), job.commitments + off * 32, (size_t)n_valid * 32);
            CUDA_TRY(cudaMemcpyAsync(l.d_commit.get(), l.h_commit.get(), (size_t)n_valid * 32, cudaMemcpyHostToDevice, stream_.get()));
            lj->commit = reinterpret_cast<const uint32_t *>(l.d_commit.get());
            lj->commit_stride = 8;
        }   // else one commitment for every item (compare jobs): only the indices travel
    }
    // rider segment [seg, n_slots): every slot gets its own commitment row and index at its layer position, whatever form
    // the rider's call had; the slots that round a chunk up to whole warps get index 0 under a zero commitment
    const uint32_t seg = p.range_slots, n_seg = p.n_slots - seg;
    if (riders) {
        bool any_cmp = false;
        for (size_t k = 0; k < p.chunks.size(); k++) {
            const RiderChunk &c = p.chunks[k];
            const Job &rj = *l.chunk_rider[k]->job;
            for (uint32_t i = 0; i < c.n; i++) {
                l.h_idx.get()[c.slot + i] = rj.indices[c.item_off + i];
                memcpy(l.h_commit.get() + (size_t)(c.slot + i) * 32, rj.row(c.item_off + i), 32);
            }
            const uint32_t pad = round_up(c.n, 32) - c.n;
            memset(l.h_idx.get() + c.slot + c.n, 0, (size_t)pad * 8);
            memset(l.h_commit.get() + (size_t)(c.slot + c.n) * 32, 0, (size_t)pad * 32);
            if (rj.expect_host) {
                memcpy(l.h_exp.get() + (size_t)c.slot * 16, rj.expect_host + c.item_off * 16, (size_t)c.n * 16);
                any_cmp = true;
            }
        }
        CUDA_TRY(cudaMemcpyAsync(l.d_idx.get() + seg, l.h_idx.get() + seg, (size_t)n_seg * 8, cudaMemcpyHostToDevice, stream_.get()));
        CUDA_TRY(cudaMemcpyAsync(l.d_commit.get() + (size_t)seg * 32, l.h_commit.get() + (size_t)seg * 32, (size_t)n_seg * 32,
                                 cudaMemcpyHostToDevice, stream_.get()));
        if (any_cmp)
            CUDA_TRY(cudaMemcpyAsync(l.d_exp.get() + (size_t)seg * 16, l.h_exp.get() + (size_t)seg * 16, (size_t)n_seg * 16,
                                     cudaMemcpyHostToDevice, stream_.get()));
    }
    if (job.gather || riders) {
        CUDA_TRY(cudaEventRecord(l.ev_in.get(), stream_.get()));
        l.in_pending = true;
    }
    CUDA_TRY(launch_pbkdf2_expand(*lj, l.X.get(), alloc_slots_, seg, stream_.get()));
    g_launches += 1;
    if (riders) {
        // K1 of the rider segment: the same kernel on the X columns from `seg` on
        const LabelJob rl{reinterpret_cast<const uint32_t *>(l.d_commit.get()) + 8 * (size_t)seg, 8, l.d_idx.get() + seg, 0, n_seg, nullptr};
        CUDA_TRY(launch_pbkdf2_expand(rl, l.X.get() + seg, alloc_slots_, n_seg, stream_.get()));
        g_launches += 1;
    }
    return B200POST_OK;
}

int DeviceEngine::finish_layer(const Job &job, int b, const LabelJob &lj) {
    Layer &l = layer_[b];
    const LayerPlan &p = l.plan;
    const uint64_t off = p.range_off;
    const uint32_t n_valid = p.n_range, n_slots = p.range_slots;
    cudaStream_t st = stream_.get();
    // the range segment (or the gather's items): K3 as without riders, so the VRF scan and cta_cand see range slots only
    if (job.expect_host) {
        // K3c: the expected slice goes H2D on the copy stream (pinned staging, double-buffered by parity; retire(b) has
        // seen the previous copy out of h_exp finish), and K3c waits for it by event
        memcpy(l.h_exp.get(), job.expect_host + off * 16, (size_t)n_valid * 16);
        CUDA_TRY(cudaMemcpyAsync(l.d_exp.get(), l.h_exp.get(), (size_t)n_valid * 16, cudaMemcpyHostToDevice, copy_stream_.get()));
        CUDA_TRY(cudaEventRecord(l.ev_exp.get(), copy_stream_.get()));
        CUDA_TRY(cudaStreamWaitEvent(st, l.ev_exp.get(), 0));
        CUDA_TRY(cudaMemsetAsync(l.d_cnt.get(), 0, 4, st));
        CUDA_TRY(launch_pbkdf2_final_compare(lj, l.X.get(), alloc_slots_, n_slots, l.d_exp.get(), l.d_bits.get(), l.d_cnt.get(),
                                           job.d_diff, d_cta_cand_.get(), st));
    } else if (job.out_hi_dev) {
        // K3w: both halves of every label32 stay in HBM (gathers of VRF-nonce checks)
        CUDA_TRY(launch_pbkdf2_final_wide(lj, l.X.get(), alloc_slots_, n_slots, job.out_dev + off * 16, job.out_hi_dev + off * 16, st));
    } else {
        uint8_t *d_out = job.out_dev ? job.out_dev + off * 16 : l.d_out.get();
        CUDA_TRY(launch_pbkdf2_final(lj, l.X.get(), alloc_slots_, n_slots, d_out, job.d_diff, d_cta_cand_.get(), st));
    }
    g_launches += 1;
    if (job.d_diff) {
        CUDA_TRY(launch_vrf_merge(d_cta_cand_.get(), pbkdf2_final_ctas(n_slots), d_running_.get(), st));
        g_launches += 1;
    }
    // the rider chunks: each one's K3 / K3w / K3c on its X columns, into the rider's own destination (a host
    // destination through d_out at the chunk's slots; a compare chunk's bitmap words and count at slot / 32)
    uint32_t copy_slots = job.out_host ? n_valid : 0;   // d_out slots the D2H takes
    bool rider_cmp = false;
    for (size_t k = 0; k < p.chunks.size(); k++) {
        const RiderChunk &c = p.chunks[k];
        const Job &rj = *l.chunk_rider[k]->job;
        const LabelJob cj{reinterpret_cast<const uint32_t *>(l.d_commit.get()) + 8 * (size_t)c.slot, 8, l.d_idx.get() + c.slot, 0, c.n, nullptr};
        const uint4 *Xc = l.X.get() + c.slot;
        if (rj.expect_host) {
            CUDA_TRY(cudaMemsetAsync(l.d_cnt.get() + c.slot / 32, 0, 4, st));
            CUDA_TRY(launch_pbkdf2_final_compare(cj, Xc, alloc_slots_, c.n, l.d_exp.get() + (size_t)c.slot * 16, l.d_bits.get() + c.slot / 32,
                                               l.d_cnt.get() + c.slot / 32, nullptr, nullptr, st));
            rider_cmp = true;
        } else if (rj.out_hi_dev) {
            CUDA_TRY(launch_pbkdf2_final_wide(cj, Xc, alloc_slots_, c.n, rj.out_dev + c.item_off * 16, rj.out_hi_dev + c.item_off * 16, st));
        } else if (rj.out_dev) {
            CUDA_TRY(launch_pbkdf2_final(cj, Xc, alloc_slots_, c.n, rj.out_dev + c.item_off * 16, nullptr, nullptr, st));
        } else {
            CUDA_TRY(launch_pbkdf2_final(cj, Xc, alloc_slots_, c.n, l.d_out.get() + (size_t)c.slot * 16, nullptr, nullptr, st));
            if (rj.out_host) copy_slots = c.slot + c.n;
        }
        g_launches += 1;
    }
    if (copy_slots || job.expect_host || rider_cmp) {
        // the copy runs on its own stream: the next layers' kernels do not queue behind PCIe.  A compare job brings
        // back only its 4-byte count (rider chunks: one per chunk, at slot / 32); the bitmap follows in retire() when it
        // is non-zero.
        CUDA_TRY(cudaEventRecord(l.ev_k3.get(), st));
        CUDA_TRY(cudaStreamWaitEvent(copy_stream_.get(), l.ev_k3.get(), 0));
        if (job.expect_host || rider_cmp)
            CUDA_TRY(cudaMemcpyAsync(l.h_cnt.get(), l.d_cnt.get(), job.expect_host ? 4 : (size_t)p.n_slots / 32 * 4, cudaMemcpyDeviceToHost,
                                     copy_stream_.get()));
        if (copy_slots)
            CUDA_TRY(cudaMemcpyAsync(l.h_out.get(), l.d_out.get(), (size_t)copy_slots * 16, cudaMemcpyDeviceToHost, copy_stream_.get()));
        CUDA_TRY(cudaEventRecord(l.ev_done.get(), copy_stream_.get()));
    } else {
        CUDA_TRY(cudaEventRecord(l.ev_done.get(), st));
    }
    l.pend.plan = p;
    l.pend.riders = l.chunk_rider;
    l.pend.live = true;
    return B200POST_OK;
}

// labels a layer's launches compute: the range segment's and the rider chunks'
static double layer_labels(const LayerPlan &p) {
    double n = p.n_range;
    for (const RiderChunk &c : p.chunks) n += c.n;
    return n;
}

int DeviceEngine::run_job(const Job &job) {
    const uint64_t S = std::min<uint64_t>(layer_labels_, alloc_slots_);
    const uint64_t M = (job.total + S - 1) / S;   // layers without riders
    int rc_ = B200POST_OK, status = B200POST_OK;
    cudaStream_t st = stream_.get();

    // small jobs (a proof's K2 labels, one VRF-nonce label, ...): the low-latency kernel, one launch
    const int64_t lowlat_max = options().lowlat_max_labels.load();
    const bool lowlat = (variant_ == ROMIX_PIPELINED || variant_ == ROMIX_PHASED) && M == 1 && lowlat_max > 0 && job.total <= (uint64_t)lowlat_max &&
                        job.total <= (uint64_t)prop_.multiProcessorCount * 4 * 32;
    // a range job that launches layers hosts riders (compare jobs do not)
    const bool host = !job.gather && !job.expect_host && !lowlat && rider_cap((uint32_t)S) > 0;
    if (host) {
        { std::lock_guard<std::mutex> lk(rider_mu_); hosting_ = true; host_N_ = job.N; }
        rider_cv_.notify_all();   // gathers waiting for the engine may ride now
    }
    uint64_t range_off = 0;   // labels (of a gather: items) of the job in the layers staged so far
    if (lowlat || variant_ != ROMIX_PIPELINED) {
        // one ROMix launch per layer: the low-latency kernel (a single layer), the phased kernel or a classic variant
        spec_.valid = false;
        for (uint64_t m = 0; range_off < job.total; m++) {
            if (job.cancel && *job.cancel) { status = B200POST_ERR_CANCELLED; break; }
            const int b = (int)(m & 1);
            Layer &l = layer_[b];
            if ((rc_ = retire(job, b))) return rc_;
            harvest(b);
            next_layer(job, range_off, S, host, l);
            range_off += l.plan.n_range;
            LabelJob lj;
            if ((rc_ = stage_layer(job, b, &lj))) return rc_;
            RomixParams rp;
            rp.V = V_; rp.X = l.X.get(); rp.x_stride = alloc_slots_; rp.N = (uint32_t)job.N;
            CUDA_TRY(cudaEventRecord(l.ev_k2a.get(), st));
            if (lowlat) {
                rp.n_slots = l.plan.n_range; rp.flags = 0;
                CUDA_TRY(launch_romix_lowlat(mw_, rp, romix_lowlat_warps(l.plan.n_range, prop_.multiProcessorCount), st));
            } else {
                rp.n_slots = l.plan.n_slots; rp.flags = (uint32_t)options().debug_skip_phase.load();
                rp.pair_offset = wave_slots_;
                CUDA_TRY(launch_romix(variant_, mw_, tpb_, rp, st));
            }
            CUDA_TRY(cudaEventRecord(l.ev_k2b.get(), st));
            l.k2_pending = true; l.k2_labels = layer_labels(l.plan);
            g_launches += 1;
            if ((rc_ = finish_layer(job, b, lj))) return rc_;
        }
    } else {
        // consume a matching speculation: layer 0 of this call was filled by the previous call's last launch
        const bool resume = !job.gather && spec_.valid && spec_.N == job.N && spec_.next_start == job.start &&
                            !memcmp(spec_.commitment, cur_commitment_, 32);
        const int poff = resume ? spec_.parity : 0;
        spec_.valid = false;
        const bool speculate = !job.gather && options().speculate_next.load() != 0 && M >= 4 && job.start + job.total + S > job.start + job.total;
        auto par = [&](uint64_t m) { return (int)((m + (uint64_t)poff) & 1); };
        LabelJob lj[2];
        bool pending_mix = false;   // the other parity holds a filled layer that this launch mixes
        int spec_parity = -1;       // parity of the speculatively filled layer
        // Each launch fills layer m (staged here) and mixes layer m-1.  Riders go only into the layers this call stages:
        // a resumed layer 0 and the speculative layer are the range job's alone.  A cancelled job still mixes and
        // finishes the layer it has filled, so that the riders in it complete.
        for (uint64_t m = 0;; m++) {
            bool more = status == B200POST_OK && range_off < job.total;
            if (more && job.cancel && *job.cancel) { status = B200POST_ERR_CANCELLED; more = false; }
            if (!more && !pending_mix) break;
            const int b = par(m);
            Layer &l = layer_[b];
            harvest(b);
            bool fill = false;
            uint32_t n_fill = 0;
            if (more) {
                if (m == 0 && resume) {
                    next_layer(job, 0, S, false, l);
                    lj[b] = LabelJob{d_range_commit_.get(), 0, nullptr, job.start, l.plan.n_range, nullptr};   // already filled: X holds its mid-state
                } else {
                    next_layer(job, range_off, S, host, l);
                    if ((rc_ = stage_layer(job, b, &lj[b]))) return rc_;
                    fill = true; n_fill = l.plan.n_slots;
                }
                range_off += l.plan.n_range;
            } else if (speculate && status == B200POST_OK) {
                // one layer past the end of this call: the next initialize() batch, if it comes
                LabelJob next;
                Job after = job;                       // the range that would follow this call: [start + total, ...)
                after.start = job.start + job.total;
                next_layer(after, 0, S, false, l);     // S labels: speculate needs M >= 4
                if ((rc_ = stage_layer(after, b, &next))) return rc_;
                fill = true; n_fill = l.plan.n_slots; spec_parity = b;
            }
            const uint32_t n_mix = pending_mix ? layer_[b ^ 1].plan.n_slots : 0;
            if (n_fill == 0 && n_mix == 0) { pending_mix = more; continue; }   // resumed call: nothing to launch for m = 0
            PipeParams pp;
            pp.V = V_; pp.x_stride = alloc_slots_; pp.N = (uint32_t)job.N;
            pp.Xfill = l.X.get(); pp.Xmix = layer_[b ^ 1].X.get();
            pp.n_fill = n_fill;
            pp.n_mix = n_mix;
            pp.fill_parity = (uint32_t)b;
            pp.cta_trace = nullptr;
            // diagnostics: B200POST_CTA_TRACE=<file> dumps {start ns, end ns, smid} per CTA of the last steady launch
            static const char *trace_path = getenv("B200POST_CTA_TRACE");
            DeviceBuffer<unsigned long long> d_trace;
            const uint32_t n_cta = (std::max(pp.n_fill, pp.n_mix) + tpb_ - 1) / tpb_;
            if (trace_path && m >= 1 && fill && more && range_off == job.total) {
                CUDA_TRY(d_trace.resize((size_t)n_cta * 3));
                CUDA_TRY(cudaMemsetAsync(d_trace.get(), 0, (size_t)n_cta * 24, st));
                pp.cta_trace = d_trace.get();
            }
            CUDA_TRY(cudaEventRecord(l.ev_k2a.get(), st));
            CUDA_TRY(launch_romix_pipe(mw_, tpb_, dr_unroll_, pp, st));
            CUDA_TRY(cudaEventRecord(l.ev_k2b.get(), st));
            l.k2_pending = true;
            l.k2_labels = 0.5 * ((fill ? layer_labels(l.plan) : 0) + (pending_mix ? layer_labels(layer_[b ^ 1].plan) : 0));
            g_launches += 1;
            if (d_trace.get()) {
                std::vector<unsigned long long> h((size_t)n_cta * 3);
                CUDA_TRY(cudaMemcpyAsync(h.data(), d_trace.get(), h.size() * 8, cudaMemcpyDeviceToHost, st));
                CUDA_TRY(cudaStreamSynchronize(st));
                if (FILE *f = fopen(trace_path, "w")) {
                    for (uint32_t c = 0; c < n_cta; c++) fprintf(f, "%u,%llu,%llu,%llu\n", c, h[3 * c], h[3 * c + 1], h[3 * c + 2]);
                    fclose(f);
                }
            }
            if (pending_mix) {
                // layer m-3 used the output buffers of this parity.  Waiting for it HERE, after launch m is queued,
                // keeps one whole launch ahead of the host: a slow wake-up, host copy or PCIe transfer does not
                // leave the GPU idle between layers.
                if ((rc_ = retire(job, b ^ 1))) return rc_;
                if ((rc_ = finish_layer(job, b ^ 1, lj[b ^ 1]))) return rc_;
            }
            pending_mix = more;
        }
        if (spec_parity >= 0 && status == B200POST_OK) {
            spec_.valid = true; spec_.N = job.N; spec_.next_start = job.start + job.total; spec_.parity = spec_parity;
            memcpy(spec_.commitment, cur_commitment_, 32);
        }
    }
    for (int b = 0; b < 2; b++) {
        Layer &l = layer_[b];
        if ((rc_ = retire(job, b))) return rc_;
        harvest(b);
        if (l.in_pending) { CUDA_TRY(cudaEventSynchronize(l.ev_in.get())); l.in_pending = false; }
    }
    return status;
}

void DeviceEngine::end_hosting(int status) {
    std::lock_guard<std::mutex> lk(rider_mu_);
    if (!hosting_) return;
    hosting_ = false;
    const bool failed = status != B200POST_OK && status != B200POST_ERR_CANCELLED;
    const std::string err = last_error();
    for (Rider *r : riders_) {
        if (failed && r->retired < r->load.placed) {
            // it had labels in a layer that did not retire: the host job's error is its error
            r->rc = status; r->err = err; r->done = true;
        } else {
            r->load.placed = r->retired;
            r->released = true;
        }
    }
    riders_.clear();
    rider_cv_.notify_all();
}

bool DeviceEngine::ride(Job &job, const std::function<int()> &setup, int *rc) {
    Rider r;
    r.load.items = job.total;
    r.job = &job;
    const auto t0 = std::chrono::steady_clock::now();
    {
        std::unique_lock<std::mutex> lk(rider_mu_);
        if (!hosting_ || host_N_ != job.N) return false;
        if (job.cmp) *job.cmp = CompareResult{};
        riders_.push_back(&r);
        rider_cv_.wait(lk, [&] { return r.done || r.released; });
    }
    const uint64_t rode = r.retired;
    if (rode == 0 && r.released) return false;   // the range job ended before any layer took it: call() goes on
    Metrics &mx = metrics();
    if (r.done) {
        *rc = r.rc;
        if (r.rc != B200POST_OK) { set_error(r.err); return true; }
        mx.gather_calls_total++;
    } else {
        // released by a range job that ended first: items [rode, total) run as an ordinary call
        Job rest = job;
        rest.total = job.total - rode;
        rest.indices += rode;
        if (rest.commitments) rest.commitments += rode * 32;
        if (rest.commit_index) rest.commit_index += rode;
        if (rest.out_host) rest.out_host += rode * 16;
        if (rest.out_dev) rest.out_dev += rode * 16;
        if (rest.out_hi_dev) rest.out_hi_dev += rode * 16;
        if (rest.expect_host) rest.expect_host += rode * 16;
        CompareResult tail;
        if (job.cmp) rest.cmp = &tail;
        *rc = call(rest, setup);
        if (job.cmp) {
            job.cmp->mismatches += tail.mismatches;
            for (uint64_t pos : tail.first)
                if (job.cmp->first.size() < CompareResult::kMaxReported) job.cmp->first.push_back(pos + rode);
        }
        if (*rc != B200POST_OK) return true;
    }
    if (!job.expect_host) mx.labels_gather_total += rode;
    mx.rider_calls_total++;
    mx.rider_labels_total += rode;
    observe_rider_wait_seconds(std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
    return true;
}

DeviceEngine::Hold::Hold(DeviceEngine &e, bool locked) : e_(e) { if (!locked) e_.mu_.lock(); }

DeviceEngine::Hold::~Hold() {
    e_.mu_.unlock();
    { std::lock_guard<std::mutex> rl(e_.rider_mu_); e_.release_gen_++; }
    e_.rider_cv_.notify_all();
}

int DeviceEngine::call(Job &job, const std::function<int()> &setup) {
    if (!job.gather || job.total == 0 || (job.cancel && *job.cancel)) {
        Hold hold(*this);
        return run_call(job, setup);
    }
    // A gather waits for the engine or for a range job it can ride, whichever comes first: one that was already waiting
    // when the range job took the engine rides it too.
    for (;;) {
        int rc = B200POST_OK;
        if (ride(job, setup, &rc)) return rc;
        uint64_t seen;
        { std::lock_guard<std::mutex> rl(rider_mu_); seen = release_gen_; }
        if (mu_.try_lock()) break;
        std::unique_lock<std::mutex> rl(rider_mu_);
        rider_cv_.wait(rl, [&] { return release_gen_ != seen || (hosting_ && host_N_ == job.N); });
    }
    Hold hold(*this, true);
    return run_call(job, setup);
}

int DeviceEngine::run_call(Job &job, const std::function<int()> &setup) {
    CUDA_TRY(cudaSetDevice(dev_));
    if (job.vrf) *job.vrf = VrfResult{};
    if (job.cmp) *job.cmp = CompareResult{};
    if (job.total == 0) return B200POST_OK;
    int rc = ensure(job.N, job.total);
    if (rc) return rc;
    cudaStream_t st = stream_.get();
    CUDA_TRY(cudaEventRecord(ev_call_[0].get(), st));
    if ((rc = setup())) return rc;
    // A cancelled job has drained what it started: like a finished one it is timed and counted, without its labels.
    const int status = run_job(job);
    if (status != B200POST_OK && status != B200POST_ERR_CANCELLED) { quiesce(); end_hosting(status); return status; }
    end_hosting(status);
    if (status == B200POST_OK && job.vrf && job.d_diff) {
        CUDA_TRY(cudaMemcpyAsync(h_running_.get(), d_running_.get(), sizeof(VrfCandidate), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        const VrfCandidate &c = *h_running_.get();
        job.vrf->found = c.found != 0;
        if (job.vrf->found) {
            job.vrf->index = c.index;
            for (int k = 0; k < 8; k++) {
                const uint32_t v = c.label_be[k];
                job.vrf->label32[4 * k] = (uint8_t)(v >> 24); job.vrf->label32[4 * k + 1] = (uint8_t)(v >> 16);
                job.vrf->label32[4 * k + 2] = (uint8_t)(v >> 8); job.vrf->label32[4 * k + 3] = (uint8_t)v;
            }
        }
    }
    CUDA_TRY(cudaEventRecord(ev_call_[1].get(), st));
    CUDA_TRY(cudaStreamSynchronize(st));
    { float ms = 0; if (cudaEventElapsedTime(&ms, ev_call_[0].get(), ev_call_[1].get()) == cudaSuccess) last_call_ms_ = ms; }
    Metrics &mx = metrics();
    (job.gather ? mx.gather_calls_total : mx.range_calls_total)++;
    mx.device_ns_total += (uint64_t)(last_call_ms_ * 1e6);
    if (status == B200POST_OK && !job.expect_host) (job.gather ? mx.labels_gather_total : mx.labels_range_total) += job.total;
    if (status == B200POST_ERR_CANCELLED) set_error("cancelled");
    return status;
}

// the commitment every item of the call shares (range and compare-indexed jobs); copied from a member, so the
// caller's buffer is free when this returns
int DeviceEngine::upload_commitment(const uint8_t commitment[32]) {
    memcpy(cur_commitment_, commitment, 32);
    CUDA_TRY(cudaMemcpyAsync(d_range_commit_.get(), cur_commitment_, 32, cudaMemcpyHostToDevice, stream_.get()));
    return B200POST_OK;
}

int DeviceEngine::labels_range(const uint8_t commitment[32], uint64_t N, uint64_t start, uint64_t count, uint8_t *out_host,
                               uint8_t *out_dev, const uint8_t *vrf_difficulty, VrfResult *vrf, const volatile int *cancel) {
    Job job;
    job.start = start; job.total = count; job.N = N; job.out_host = out_host; job.out_dev = out_dev; job.vrf = vrf; job.cancel = cancel;
    return range_call(job, commitment, vrf_difficulty);
}

int DeviceEngine::labels_compare_range(const uint8_t commitment[32], uint64_t N, uint64_t start, uint64_t count,
                                       const uint8_t *expect_host, const uint8_t *vrf_difficulty, VrfResult *vrf,
                                       CompareResult *cmp, const volatile int *cancel) {
    if (!expect_host || !cmp) { set_error("compare job without expected labels or result"); return B200POST_ERR_INVALID_ARGUMENT; }
    Job job;
    job.start = start; job.total = count; job.N = N; job.expect_host = expect_host; job.cmp = cmp; job.vrf = vrf; job.cancel = cancel;
    return range_call(job, commitment, vrf_difficulty);
}

// per-call constants of a range job: commitment, VRF threshold, running candidate
int DeviceEngine::range_call(Job &job, const uint8_t commitment[32], const uint8_t *vrf_difficulty) {
    return call(job, [&]() -> int {
        const int rc = upload_commitment(commitment);
        if (rc || !vrf_difficulty) return rc;
        uint32_t be[8];
        for (int k = 0; k < 8; k++)
            be[k] = ((uint32_t)vrf_difficulty[4 * k] << 24) | ((uint32_t)vrf_difficulty[4 * k + 1] << 16) |
                    ((uint32_t)vrf_difficulty[4 * k + 2] << 8) | vrf_difficulty[4 * k + 3];
        CUDA_TRY(cudaMemcpyAsync(d_diff_.get(), be, 32, cudaMemcpyHostToDevice, stream_.get()));
        CUDA_TRY(cudaMemsetAsync(d_running_.get(), 0, sizeof(VrfCandidate), stream_.get()));
        CUDA_TRY(cudaStreamSynchronize(stream_.get()));   // `be` is a stack buffer
        job.d_diff = d_diff_.get();
        return B200POST_OK;
    });
}

int DeviceEngine::labels_gather(size_t n_items, const uint8_t *commitments, const uint64_t *indices, uint64_t N, uint8_t *out_host,
                                uint8_t *out_dev) {
    Job job;
    job.gather = true; job.commitments = commitments; job.indices = indices; job.total = n_items; job.N = N;
    job.out_host = out_host; job.out_dev = out_dev;
    return call(job, []() -> int { return B200POST_OK; });
}

int DeviceEngine::labels_gather_indexed(size_t n_items, size_t n_commit, const uint8_t *commitments, const uint32_t *commit_index,
                                        const uint64_t *indices, uint64_t N, uint8_t *out_host, uint8_t *out_dev,
                                        uint8_t *out_hi_dev) {
    if (out_hi_dev && (!out_dev || out_host)) { set_error("out_hi_dev needs out_dev (and no out_host)"); return B200POST_ERR_INVALID_ARGUMENT; }
    for (size_t i = 0; commit_index && i < n_items; i++)
        if (commit_index[i] >= n_commit) { set_error("commitment row index past the commitment table"); return B200POST_ERR_INVALID_ARGUMENT; }
    Job job;
    job.gather = true; job.commit_table = commitments; job.commit_index = commit_index; job.indices = indices; job.total = n_items; job.N = N;
    job.out_host = out_host; job.out_dev = out_dev; job.out_hi_dev = out_hi_dev;
    return call(job, [&]() -> int {
        CUDA_TRY(d_ctab_.grow(n_commit * 32));
        CUDA_TRY(cudaMemcpyAsync(d_ctab_.get(), commitments, n_commit * 32, cudaMemcpyHostToDevice, stream_.get()));
        return B200POST_OK;
    });
}

int DeviceEngine::labels_compare_indexed(const uint8_t commitment[32], size_t n_items, const uint64_t *indices, uint64_t N,
                                         const uint8_t *expect_host, CompareResult *cmp, const volatile int *cancel) {
    if (!commitment || !indices || !expect_host || !cmp) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    Job job;
    job.gather = true; job.commit_table = commitment; job.indices = indices; job.total = n_items; job.N = N; job.expect_host = expect_host;
    job.cmp = cmp;
    job.cancel = cancel;
    return call(job, [&] { return upload_commitment(commitment); });
}

// After a failed job: drain the stream and forget every in-flight buffer, so that the next call starts clean
// (the error text of the failure is preserved).
void DeviceEngine::quiesce() {
    const std::string keep = last_error();
    if (stream_.get()) cudaStreamSynchronize(stream_.get());
    if (copy_stream_.get()) cudaStreamSynchronize(copy_stream_.get());
    cudaGetLastError();
    for (Layer &l : layer_) { l.pend.live = false; l.pend.riders.clear(); l.k2_pending = false; l.in_pending = false; }
    spec_.valid = false;
    set_error(keep);
}

uint32_t DeviceEngine::wave_slots(uint64_t N) {
    Hold lk(*this);
    if (cudaSetDevice(dev_) != cudaSuccess) return 0;
    if (ensure(N, 32) != B200POST_OK) return 0;
    return wave_slots_;
}

int DeviceEngine::timer_mark(int which) {
    Hold lk(*this);
    CUDA_TRY(cudaSetDevice(dev_));
    if (which < 0 || which > 1) return B200POST_ERR_INVALID_ARGUMENT;
    if (!stream_.get()) { int rc = ensure(2, 32); if (rc) return rc; }
    if (!ev_timer_[which].get()) CUDA_TRY(ev_timer_[which].create(cudaEventDefault));
    CUDA_TRY(cudaEventRecord(ev_timer_[which].get(), stream_.get()));
    return B200POST_OK;
}

double DeviceEngine::timer_elapsed_ms() {
    Hold lk(*this);
    if (!ev_timer_[0].get() || !ev_timer_[1].get() || cudaSetDevice(dev_) != cudaSuccess) return -1.0;
    float ms = 0;
    if (cudaEventSynchronize(ev_timer_[1].get()) != cudaSuccess || cudaEventElapsedTime(&ms, ev_timer_[0].get(), ev_timer_[1].get()) != cudaSuccess) return -1.0;
    return ms;
}

double DeviceEngine::last_call_ms() {
    Hold lk(*this);
    return last_call_ms_;
}

void DeviceEngine::romix_time(double *ms_total, uint64_t *launches, double *labels, bool reset) {
    Hold lk(*this);
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

int provider_devices(int64_t provider_id, std::vector<uint32_t> *devs) {
    if (provider_id == (int64_t)B200POST_CPU_PROVIDER_ID) return fail(B200POST_ERR_UNSUPPORTED, "provider 0xffffffff (CPU): this library has no CPU path");
    const int n = device_count();
    if (n == 0) return fail(B200POST_ERR_NO_DEVICE, "no CUDA device available");
    if (provider_id != B200POST_PROVIDER_ALL) devs->push_back((uint32_t)provider_id);
    else for (int d = 0; d < n; d++) devs->push_back((uint32_t)d);
    return B200POST_OK;
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

int device_engine(uint32_t provider, DeviceEngine **e) {
    DeviceEngine *got = engine_for(provider);
    if (e) *e = got;
    if (got) return B200POST_OK;
    return provider == B200POST_CPU_PROVIDER_ID ? B200POST_ERR_UNSUPPORTED : B200POST_ERR_NO_DEVICE;
}

int device_engines(const uint32_t *providers, int n, std::vector<DeviceEngine *> *out) {
    if (out) out->assign((size_t)n, nullptr);
    for (int i = 0; i < n; i++)
        if (int rc = device_engine(providers[i], out ? &(*out)[(size_t)i] : nullptr)) return rc;
    return B200POST_OK;
}

void shutdown_all() {
    std::lock_guard<std::mutex> lk(g_reg_mu);
    g_engines.clear();
}

int fan_out(size_t parts, const std::function<int(size_t)> &part) {
    std::vector<int> rcs(parts, B200POST_OK);
    std::vector<std::string> errs(parts);
    std::vector<std::thread> th;
    for (size_t i = 0; i < parts; i++)
        th.emplace_back([&, i] {
            if ((rcs[i] = part(i)) != B200POST_OK) errs[i] = last_error();
        });
    for (auto &t : th) t.join();
    for (size_t i = 0; i < parts; i++)
        if (rcs[i] != B200POST_OK) return fail(rcs[i], errs[i]);
    return B200POST_OK;
}

int label32_at(DeviceEngine *e, const uint8_t commitment[32], uint64_t N, uint64_t index, uint8_t out[32]) {
    uint8_t all[32];
    memset(all, 0xff, 32);
    VrfResult vr;
    if (int rc = e->labels_range(commitment, N, index, 1, nullptr, nullptr, all, &vr, nullptr)) return rc;
    if (!vr.found) memset(vr.label32, 0xff, 32);   // found is 0 only for the all-ones label
    memcpy(out, vr.label32, 32);
    return B200POST_OK;
}

}  // namespace b200post
