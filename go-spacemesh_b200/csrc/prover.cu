// prover.cu — POST proof generation scan (include/b200post_prove.h, SURVEY.md §8f.3).
//
// K6 prove_scan_kernel streams 16-byte labels (H2D from the postdata files, double-buffered) through one
// AES-128 cipher per nonce group and appends (nonce, index) hits to a small list; the host keeps the per-nonce
// hit lists and stops when a nonce owns K2 of them.  Bandwidth view: 16 B in per label, ~nothing out; the
// kernel is far faster than PCIe/NVMe can feed it, so the design goal is simply to keep copies and compute
// overlapped.  Conventions: post-rs Prover8_56 from memory (ASSUMED, unpinned).
//
// Several devices (b200post_generate_proof_multi): the label range is split into contiguous shards, one host thread and
// Scanner each; their hit lists merge in shard order (ShardedScan), so the proof is the one-device proof.
//
// Damaged stored data (b200post_generate_proof_checked): the kernels also return each hit's stored bytes (StoredHit), and
// the stop rule's tentative winner has its first K2 hits recomputed and compared on the device before the scan may stop
// on it; damaged hits are dropped (DESIGN.md §5).
//
// Nonce windows (b200post_prove_opts.max_windows): generate() runs passes over the data, each scanning windows_per_pass
// windows of nonces with their own pows, until a window has a proof; the kernels only ever see pass-relative nonces.
//
// The scanner, the selection rule, the proof record, the pow step and the verifier gate are declared in prove_internal.h:
// the setup session's initial proof (initial_proof.cu) runs the same scan over the labels as it writes them.
#include <algorithm>
#include <atomic>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <thread>
#include <vector>

#include "../../include/b200post_prove.h"
#include "../../include/b200post_k2pow.h"
#include "aes_device.cuh"
#include "engine.h"
#include "metrics.h"
#include "postdata_io.h"
#include "proof_common.h"
#include "prove_internal.h"

namespace b200post {
namespace {

struct Hit { uint32_t nonce; uint32_t pad; uint64_t index; };
// b200post_generate_proof_checked's record: the hit and the 16 stored bytes the kernel judged
struct StoredHit { uint32_t nonce; uint32_t pad; uint64_t index; uint4 label; };

__device__ __forceinline__ Hit make_hit(const Hit *, uint32_t nonce, uint64_t index, uint4) { return Hit{nonce, 0, index}; }
__device__ __forceinline__ StoredHit make_hit(const StoredHit *, uint32_t nonce, uint64_t index, uint4 label) {
    return StoredHit{nonce, 0, index, label};
}

// K6a: rk = per nonce group 11 round keys.  Every (label, group) costs one AES; ciphertext bytes below the
// difficulty MSB are hits, bytes EQUAL to it (1 in 256) need the nonce's "lazy" cipher: those are queued as
// (label offset, nonce) candidates and resolved densely by K6b — evaluating them in place would run a whole
// AES with one or two active lanes for most warps.  Rec = Hit, or StoredHit to keep the label bytes with the hit.
template <class Rec>
__global__ void __launch_bounds__(256) prove_scan_kernel(const uint4 *__restrict__ labels, uint64_t first_index, uint32_t count,
                                                         const uint4 *__restrict__ rk, uint32_t n_groups, uint32_t diff_msb,
                                                         const AesTables *__restrict__ tables, Rec *__restrict__ hits,
                                                         uint32_t hit_cap, uint32_t *__restrict__ n_hits,
                                                         uint2 *__restrict__ cands, uint32_t cand_cap, uint32_t *__restrict__ n_cands) {
    extern __shared__ uint32_t aes_sm[];
    aes_load_smem(aes_sm, tables);
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t *tl = aes_sm + lane;
    const uint32_t msb4 = diff_msb * 0x01010101u;
    const uint32_t stride = gridDim.x * blockDim.x;
    // whole warps stay in the loop together (the candidate compaction below is warp-collective)
    for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) - lane; base < count; base += stride) {
        const uint32_t i = base + lane;
        const bool live = i < count;
        const uint4 label = live ? labels[i] : make_uint4(0, 0, 0, 0);
        for (uint32_t g = 0; g < n_groups; g++) {
            const uint4 out = aes128_encrypt(tl, rk + 11 * g, label);
            // per byte: 0xff where ciphertext byte <= MSB / == MSB
            const uint32_t le[4] = {__vcmpleu4(out.x, msb4), __vcmpleu4(out.y, msb4), __vcmpleu4(out.z, msb4), __vcmpleu4(out.w, msb4)};
            const uint32_t eq[4] = {__vcmpeq4(out.x, msb4), __vcmpeq4(out.y, msb4), __vcmpeq4(out.z, msb4), __vcmpeq4(out.w, msb4)};
            const bool any_le = live && (le[0] | le[1] | le[2] | le[3]);
            if (!__any_sync(0xffffffffu, any_le)) continue;
            uint32_t n_eq = 0;
            if (any_le) {
#pragma unroll
                for (int w = 0; w < 4; w++) n_eq += __popc(eq[w]) >> 3;
            }
            // warp-aggregated reservation of candidate slots
            uint32_t incl = n_eq;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (uint32_t)d) incl += t; }
            const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
            uint32_t slot = 0;
            if (total) {
                if (lane == 31) slot = atomicAdd(n_cands, total);
                slot = __shfl_sync(0xffffffffu, slot, 31) + incl - n_eq;
            }
            if (any_le) {
#pragma unroll 1
                for (uint32_t b = 0; b < 16; b++) {
                    const uint32_t bit = 0xffu << (8 * (b & 3));
                    if (!(le[b >> 2] & bit)) continue;
                    const uint32_t nonce = g * 16 + b;
                    if (eq[b >> 2] & bit) {
                        if (slot < cand_cap) cands[slot] = make_uint2(i, nonce);
                        slot++;
                    } else {
                        const uint32_t pos = atomicAdd(n_hits, 1u);
                        if (pos < hit_cap) hits[pos] = make_hit(hits, nonce, first_index + i, label);
                    }
                }
            }
        }
    }
}

// K6b: one thread per candidate: the nonce's lazy cipher decides with the low 56 bits.
template <class Rec>
__global__ void __launch_bounds__(256) prove_lazy_kernel(const uint4 *__restrict__ labels, uint64_t first_index,
                                                         const uint2 *__restrict__ cands, const uint32_t *__restrict__ n_cands,
                                                         uint32_t cand_cap, const uint4 *__restrict__ lazy_rk, uint64_t diff_lsb,
                                                         const AesTables *__restrict__ tables, Rec *__restrict__ hits,
                                                         uint32_t hit_cap, uint32_t *__restrict__ n_hits) {
    extern __shared__ uint32_t aes_sm[];
    aes_load_smem(aes_sm, tables);
    const uint32_t *tl = aes_sm + (threadIdx.x & 31);
    const uint32_t n = min(*n_cands, cand_cap);
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const uint2 cd = cands[c];
        const uint4 label = labels[cd.x];
        const uint4 lz = aes128_encrypt(tl, lazy_rk + 11 * cd.y, label);
        const uint64_t lsb = ((uint64_t)lz.x | ((uint64_t)lz.y << 32)) & 0x00ffffffffffffffull;
        if (lsb >= diff_lsb) continue;
        const uint32_t pos = atomicAdd(n_hits, 1u);
        if (pos < hit_cap) hits[pos] = make_hit(hits, cd.y, first_index + cd.x, label);
    }
}

}  // namespace

bool pick_winner_in(const HitLists &lists, uint32_t lo, uint32_t hi, uint32_t k2, uint32_t *nonce, std::vector<uint64_t> *indices) {
    bool have = false;
    for (auto it = lists.lower_bound(lo); it != lists.end() && it->first < hi; ++it) {
        if (it->second.size() < k2) continue;
        if (!have || it->second[k2 - 1] < (*indices)[k2 - 1]) { *nonce = it->first; *indices = it->second; have = true; }
    }
    return have;
}

bool pick_winner(const HitLists &lists, uint32_t k2, uint32_t *nonce, std::vector<uint64_t> *indices) {
    return pick_winner_in(lists, 0, UINT32_MAX, k2, nonce, indices);
}

int Scanner::init(uint32_t provider, const uint8_t challenge[32], uint32_t nonces, const uint64_t *pows, uint32_t k1, uint32_t k2,
                  uint64_t num_labels, uint64_t chunk, bool keep_stored, uint32_t first_nonce) {
    DeviceEngine *e = engine_for(provider);
    if (!e) return provider == B200POST_CPU_PROVIDER_ID ? B200POST_ERR_UNSUPPORTED : B200POST_ERR_NO_DEVICE;
    if (nonces == 0 || nonces % 16 || first_nonce % 16 || (uint64_t)first_nonce + nonces > 4096 || k1 == 0 || k2 == 0 ||
        num_labels == 0 || chunk == 0 || chunk > (1u << 28)) {
        set_error("invalid proving parameters (nonces must be a positive multiple of 16, <= 4096)");
        return B200POST_ERR_INVALID_ARGUMENT;
    }
    engine_ = e; dev_ = e->device(); nonces_ = nonces; first_ = first_nonce; k2_ = k2; chunk_ = chunk;
    stored_ = keep_stored; rec_ = stored_ ? sizeof(StoredHit) : sizeof(Hit);
    const uint64_t diff = b200post_proving_difficulty(k1, num_labels);
    msb_ = (uint32_t)(diff >> 56); lsb_ = diff & 0x00ffffffffffffffull;
    // hits per chunk are ~ chunk * nonces * K1/numLabels; leave generous slack, cap the buffer at 64 MiB
    const double expect = (double)chunk * nonces * ((double)k1 / (double)num_labels);
    hit_cap_ = (uint32_t)std::min<double>(std::max<double>(4.0 * expect + 65536.0, 65536.0), 4.0 * 1024 * 1024);
    CUDA_TRY(cudaSetDevice(dev_));
    std::vector<uint8_t> rk((size_t)(nonces / 16) * 176), lazy((size_t)nonces * 176);
    // keys of the absolute groups and nonces; the kernels index them from 0, so their hit nonces are pass-relative
    for (uint32_t g = 0; g < nonces / 16; g++) {
        uint8_t key[16];
        cipher_key(challenge, first_nonce / 16 + g, pows[g], nullptr, key);
        const Aes128 a(key);
        memcpy(rk.data() + (size_t)g * 176, a.rk, 176);
    }
    for (uint32_t n = 0; n < nonces; n++) {
        uint8_t key[16];
        const uint32_t abs = first_nonce + n;
        cipher_key(challenge, abs / 16, pows[n / 16], &abs, key);
        const Aes128 a(key);
        memcpy(lazy.data() + (size_t)n * 176, a.rk, 176);
    }
    static AesTables host_tables;
    static std::once_flag once;
    std::call_once(once, [] { aes_build_tables(host_tables); });
    CUDA_TRY(d_rk_.resize(rk.size()));
    CUDA_TRY(d_lazy_.resize(lazy.size()));
    CUDA_TRY(d_tables_.resize(1));
    CUDA_TRY(cudaMemcpy(d_rk_.get(), rk.data(), rk.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(d_lazy_.get(), lazy.data(), lazy.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(d_tables_.get(), &host_tables, sizeof(AesTables), cudaMemcpyHostToDevice));
    for (int b = 0; b < 2; b++) {
        CUDA_TRY(st_[b].create(cudaStreamNonBlocking));
        CUDA_TRY(ev_[b].create(cudaEventDisableTiming));
        CUDA_TRY(d_labels_[b].resize(chunk * 16));
        CUDA_TRY(h_labels_[b].resize(chunk * 16));
        CUDA_TRY(d_hits_[b].resize((size_t)hit_cap_ * rec_));
        CUDA_TRY(d_nhits_[b].resize(1));
        CUDA_TRY(h_hits_[b].resize((size_t)hit_cap_ * rec_));
        CUDA_TRY(h_nhits_[b].resize(1));
        CUDA_TRY(h_ncands_[b].resize(1));
    }
    // lazy-cipher candidates: one ciphertext byte in 256 equals the MSB; 2x slack, shared by both buffers
    // (chunks are processed in stream order on alternating streams, so the queue is fenced by events below)
    cand_cap_ = (uint32_t)std::min<uint64_t>((chunk * nonces) / 128 + 65536, 1u << 27);
    CUDA_TRY(d_cands_.resize(cand_cap_));
    CUDA_TRY(d_ncands_.resize(2));
    cudaDeviceProp p;
    CUDA_TRY(cudaGetDeviceProperties(&p, dev_));
    grid_ = (uint32_t)p.multiProcessorCount * 6;   // 6 CTAs x 32 KiB of lane-replicated AES table per SM
    return B200POST_OK;
}

template <class Rec>
void Scanner::launch(cudaStream_t st, const uint4 *labels, uint64_t first, uint32_t count, Rec *hits, uint32_t *n_hits) {
    prove_scan_kernel<Rec><<<grid_, 256, AES_SMEM_BYTES, st>>>(labels, first, count, reinterpret_cast<const uint4 *>(d_rk_.get()), nonces_ / 16,
                                                               msb_, d_tables_.get(), hits, hit_cap_, n_hits, d_cands_.get(), cand_cap_,
                                                               d_ncands_.get());
    prove_lazy_kernel<Rec><<<grid_, 256, AES_SMEM_BYTES, st>>>(labels, first, d_cands_.get(), d_ncands_.get(), cand_cap_,
                                                               reinterpret_cast<const uint4 *>(d_lazy_.get()), lsb_, d_tables_.get(),
                                                               hits, hit_cap_, n_hits);
}

int Scanner::submit(int b, uint64_t first, uint32_t count) {
    CUDA_TRY(cudaMemcpyAsync(d_labels_[b].get(), h_labels_[b].get(), (size_t)count * 16, cudaMemcpyHostToDevice, st_[b].get()));
    CUDA_TRY(cudaMemsetAsync(d_nhits_[b].get(), 0, 4, st_[b].get()));
    // the single candidate queue is reused by consecutive chunks: wait for the other stream's lazy pass
    if (pending_[b ^ 1]) CUDA_TRY(cudaStreamWaitEvent(st_[b].get(), ev_[b ^ 1].get(), 0));
    CUDA_TRY(cudaMemsetAsync(d_ncands_.get(), 0, 8, st_[b].get()));
    cudaStream_t st = st_[b].get();
    const uint4 *labels = reinterpret_cast<const uint4 *>(d_labels_[b].get());
    if (stored_) launch(st, labels, first, count, reinterpret_cast<StoredHit *>(d_hits_[b].get()), d_nhits_[b].get());
    else launch(st, labels, first, count, reinterpret_cast<Hit *>(d_hits_[b].get()), d_nhits_[b].get());
    g_launches += 2;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(h_ncands_[b].get(), d_ncands_.get(), 4, cudaMemcpyDeviceToHost, st_[b].get()));
    CUDA_TRY(cudaMemcpyAsync(h_nhits_[b].get(), d_nhits_[b].get(), 4, cudaMemcpyDeviceToHost, st_[b].get()));
    CUDA_TRY(cudaMemcpyAsync(h_hits_[b].get(), d_hits_[b].get(), (size_t)hit_cap_ * rec_, cudaMemcpyDeviceToHost, st_[b].get()));
    CUDA_TRY(cudaEventRecord(ev_[b].get(), st_[b].get()));
    pending_[b] = true; count_[b] = count;
    return B200POST_OK;
}

int Scanner::collect(int b, std::mutex *fold_mu) {
    if (!pending_[b]) return B200POST_OK;
    CUDA_TRY(cudaEventSynchronize(ev_[b].get()));
    pending_[b] = false;
    const uint32_t n = *h_nhits_[b].get();
    if (n > hit_cap_ || *h_ncands_[b].get() > cand_cap_) { set_error("hit buffer overflow: K1 too large for this chunk size"); return B200POST_ERR_OUT_OF_MEMORY; }
    if (stored_) return fold_stored(b, n, fold_mu);
    const Hit *rec = reinterpret_cast<const Hit *>(h_hits_[b].get());
    std::vector<Hit> v(rec, rec + n);
    std::sort(v.begin(), v.end(), [](const Hit &x, const Hit &y) { return x.index != y.index ? x.index < y.index : x.nonce < y.nonce; });
    std::unique_lock<std::mutex> lk;
    if (fold_mu) lk = std::unique_lock<std::mutex>(*fold_mu);
    for (const Hit &h : v) {
        std::vector<uint64_t> &l = lists_[first_ + h.nonce];
        if (l.size() < k2_ && (l.push_back(h.index), l.size() == k2_)) full_++;
    }
    scanned_ += count_[b];   // chunks are contiguous from the first index: the sum is how far the scan went
    return B200POST_OK;
}

int Scanner::fold_stored(int b, uint32_t n, std::mutex *fold_mu) {
    const StoredHit *rec = reinterpret_cast<const StoredHit *>(h_hits_[b].get());
    std::vector<StoredHit> v(rec, rec + n);
    std::sort(v.begin(), v.end(), [](const StoredHit &x, const StoredHit &y) { return x.index != y.index ? x.index < y.index : x.nonce < y.nonce; });
    std::unique_lock<std::mutex> lk;
    if (fold_mu) lk = std::unique_lock<std::mutex>(*fold_mu);
    for (const StoredHit &h : v) {
        KeptHit k{h.index, {}, false};
        memcpy(k.label, &h.label, 16);
        kept_[first_ + h.nonce].push_back(k);
    }
    scanned_ += count_[b];
    return B200POST_OK;
}

void Scanner::drain() {
    for (int b = 0; b < 2; b++) if (pending_[b]) { cudaEventSynchronize(ev_[b].get()); pending_[b] = false; }
}

void Scanner::restore(const HitLists &lists) {
    lists_ = lists;
    full_ = 0;
    for (const auto &kv : lists_) full_ += kv.second.size() >= k2_;
}

uint32_t Scanner::count_kept(bool good_only) const {
    uint32_t full = 0;
    for (const auto &kv : kept_) {
        size_t c = 0;
        for (const KeptHit &k : kv.second) if ((c += !good_only || k.good) >= k2_) break;
        full += c >= k2_;
    }
    return full;
}

namespace {

// One contiguous label range [lo, hi) of a scan, streamed through its own Scanner.
struct Shard {
    Scanner sc;
    uint64_t lo = 0, hi = 0;
    int rc = B200POST_OK;
    std::string err;
};

// The labels [0, total) in contiguous shards of whole chunks, one per provider in list order, sized within one chunk of
// each other (the earlier shards take the odd chunks; a shard may be empty).
std::vector<std::pair<uint64_t, uint64_t>> split_shards(uint64_t total, uint64_t chunk, size_t n) {
    const uint64_t chunks = (total + chunk - 1) / chunk, q = chunks / n, r = chunks % n;
    std::vector<std::pair<uint64_t, uint64_t>> out(n);
    for (size_t s = 0; s < n; s++) {
        const uint64_t first = s * q + std::min<uint64_t>(s, r), end = first + q + (s < r ? 1 : 0);
        out[s] = {std::min(total, first * chunk), std::min(total, end * chunk)};
    }
    return out;
}

// A scan split into shards, one host thread each.  Stop rule: let x be the end of the longest gap-free scanned prefix
// of [0, total), where a saturated shard counts as whole.  Once the hits below x give some nonce K2 of them the proof is
// decided (every hit below x is known, so no nonce whose K2-th hit lies past x can win) and every shard stops.  A shard
// also stops on its own once it is saturated.  With one shard this is "stop once a nonce has K2 hits".
// One pass of a windowed proof scans `windows` nonce windows of `window` nonces from nonce `first`; the stop rule then
// looks at the pass's lowest window only, saturation at every nonce of the pass, and the decision walks the windows in
// order (DESIGN.md §5).
class ShardedScan {
public:
    // fill(shard, first label, count, dst): those labels into the shard's pinned staging
    using Fill = std::function<int(size_t, uint64_t, uint64_t, uint8_t *)>;

    ShardedScan(size_t n, uint32_t first, uint32_t window, uint32_t windows, uint32_t k2)
        : first_(first), window_(window), windows_(windows), k2_(k2) {
        for (size_t s = 0; s < n; s++) shards_.emplace_back(new Shard);
    }
    Shard &shard(size_t s) { return *shards_[s]; }

    // After run() (unchecked): the winner of the lowest window of the pass that has one, over merged()
    bool winner(uint32_t *nonce, std::vector<uint64_t> *indices) const {
        const HitLists m = merged();
        for (uint32_t w = 0; w < windows_; w++)
            if (pick_winner_in(m, lo(w), lo(w) + window_, k2_, nonce, indices)) return true;
        return false;
    }

    // runs every shard (the calling thread alone when there is one) and returns the first failing shard's status, in
    // list order, once every thread has joined
    int run(const Fill &fill, uint64_t chunk, uint64_t base, const volatile int *cancel) {
        if (shards_.size() == 1) return run_shard(0, fill, chunk, base, cancel);
        std::vector<std::thread> th;
        for (size_t s = 0; s < shards_.size(); s++)
            th.emplace_back([&, s] {
                Shard &sh = *shards_[s];
                if ((sh.rc = run_shard(s, fill, chunk, base, cancel)) != B200POST_OK) { sh.err = last_error(); abort_ = true; }
            });
        for (auto &t : th) t.join();
        for (auto &sh : shards_) if (sh->rc != B200POST_OK) { set_error(sh->err); return sh->rc; }
        return B200POST_OK;
    }

    // per nonce, the shards' hit lists appended in shard order, first K2 kept; with the stop rule above, the winner of
    // these lists is the winner of a scan over every label
    HitLists merged() const {
        HitLists m;
        for (const auto &sh : shards_)
            for (const auto &kv : sh->sc.lists()) {
                std::vector<uint64_t> &l = m[kv.first];
                for (size_t i = 0; i < kv.second.size() && l.size() < k2_; i++) l.push_back(kv.second[i]);
            }
        return m;
    }
    uint64_t scanned() const {
        uint64_t t = 0;
        for (const auto &sh : shards_) t += sh->sc.scanned();
        return t;
    }

    // ---- the checked proof (b200post_generate_proof_checked): every hit is kept with its stored bytes, and the stop
    // rule's tentative winner has its first K2 hits recomputed under `commitment` before the scan may stop on it
    void enable_check(const uint8_t commitment[32], uint64_t N, const volatile int *cancel) {
        checked_ = true;
        memcpy(commitment_, commitment, 32);
        N_ = N; cancel_ = cancel;
    }
    // After run(): per window of the pass in order, recheck rounds over everything kept until the window's winner has
    // its first K2 hits all good (the winner and its indices) or no nonce of it has K2 usable hits (the next window);
    // false with *rc OK when no window has one.  Needs no round when the scan stopped on a decision.
    bool decide(uint32_t *nonce, std::vector<uint64_t> *indices, int *rc) {
        *rc = B200POST_OK;
        for (uint32_t w = 0; w < windows_; w++)
            for (;;) {
                std::vector<Item> items;
                const Plan p = plan_winner(w, &items, nonce, indices);
                if (p == DECIDED) return true;
                if (p == NONE) break;
                if ((*rc = round(shards_[0]->sc.engine(), items))) return false;
            }
        return false;
    }
    uint64_t rechecked() const { return rechecked_; }
    uint32_t rounds() const { return rounds_; }
    const std::set<uint64_t> &damaged() const { return damaged_; }

private:
    struct Item { size_t shard; uint32_t nonce; uint64_t index; uint8_t label[16]; };
    enum Plan { NONE, DECIDED, RECHECK };

    uint32_t lo(uint32_t w) const { return first_ + w * window_; }   // the first nonce of window w of the pass

    // Under mu_ (or with the threads joined).  The stop rule over kept (good and pending) hits below x of the nonces of
    // window w of the pass: NONE if no such nonce has K2 of them; DECIDED with the winner when the winner's first K2 are
    // all good; RECHECK with the pending ones.
    Plan plan_winner(uint32_t w, std::vector<Item> *items, uint32_t *nonce, std::vector<uint64_t> *indices) const {
        struct Ref { size_t shard; const KeptHit *k; };
        std::map<uint32_t, std::vector<Ref>> m;   // per nonce, its first K2 kept hits below x in shard order
        for (size_t s = 0; s < shards_.size(); s++) {
            const Scanner &sc = shards_[s]->sc;
            for (auto kv = sc.kept().lower_bound(lo(w)); kv != sc.kept().end() && kv->first < lo(w) + window_; ++kv) {
                std::vector<Ref> &l = m[kv->first];
                for (size_t i = 0; i < kv->second.size() && l.size() < k2_; i++) l.push_back({s, &kv->second[i]});
            }
            if (sc.scanned() < shards_[s]->hi - shards_[s]->lo && !sc.saturated()) break;   // x lies in this shard
        }
        const std::pair<const uint32_t, std::vector<Ref>> *win = nullptr;
        for (const auto &kv : m)
            if (kv.second.size() >= k2_ && (!win || kv.second[k2_ - 1].k->index < win->second[k2_ - 1].k->index)) win = &kv;
        if (!win) return NONE;
        for (const Ref &r : win->second) {
            if (r.k->good) continue;
            Item it{r.shard, win->first, r.k->index, {}};
            memcpy(it.label, r.k->label, 16);
            items->push_back(it);
        }
        if (!items->empty()) return RECHECK;
        *nonce = win->first;
        indices->clear();
        for (const Ref &r : win->second) indices->push_back(r.k->index);
        return DECIDED;
    }
    // Under mu_: when every nonce has K2 kept hits in shard s but not K2 good ones, the pending ones among each nonce's
    // first K2 in the shard (the shard's own saturation stop counts good hits only).
    bool plan_saturation(size_t s, std::vector<Item> *items) const {
        const Scanner &sc = shards_[s]->sc;
        if (sc.count_kept(false) != sc.nonces()) return false;
        for (const auto &kv : sc.kept())
            for (size_t i = 0; i < kv.second.size() && i < k2_; i++) {
                const KeptHit &k = kv.second[i];
                if (k.good) continue;
                Item it{s, kv.first, k.index, {}};
                memcpy(it.label, k.label, 16);
                items->push_back(it);
            }
        return !items->empty();
    }
    // One recheck round on `e` (outside mu_): the items' labels recomputed and compared with their stored bytes, then,
    // under mu_ when threads run, good ones marked and damaged ones dropped.  A compare reports at most
    // CompareResult::kMaxReported positions, so it is repeated past the last reported one until every mismatch is known.
    int round(DeviceEngine *e, const std::vector<Item> &items) {
        const size_t n = items.size();
        std::vector<uint64_t> idx(n);
        std::vector<uint8_t> expect(n * 16), bad(n, 0);
        for (size_t i = 0; i < n; i++) { idx[i] = items[i].index; memcpy(&expect[i * 16], items[i].label, 16); }
        for (size_t from = 0; from < n;) {
            CompareResult cmp;
            const int rc = e->labels_compare_indexed(commitment_, n - from, idx.data() + from, N_, expect.data() + from * 16, &cmp, cancel_);
            if (rc) return rc;
            for (uint64_t p : cmp.first) bad[from + p] = 1;
            if (cmp.mismatches <= cmp.first.size()) break;
            from += cmp.first.back() + 1;
        }
        std::unique_lock<std::mutex> lk(mu_);
        for (size_t i = 0; i < n; i++) {
            std::vector<KeptHit> &l = shards_[items[i].shard]->sc.kept()[items[i].nonce];
            auto it = std::lower_bound(l.begin(), l.end(), items[i].index, [](const KeptHit &k, uint64_t v) { return k.index < v; });
            if (it == l.end() || it->index != items[i].index) continue;
            if (bad[i]) { l.erase(it); damaged_.insert(items[i].index); }
            else it->good = true;
        }
        rechecked_ += n; rounds_++;
        return B200POST_OK;
    }
    // The checked stop rule for shard s, run by its thread after each chunk: stop once a decision is taken or the shard is
    // saturated by good hits.  When the multi-device stop rule fires (or the shard would saturate) this thread runs recheck
    // rounds until that settles, while the other shards keep scanning.  One winner round runs at a time; a saturation
    // round touches only its own shard's hits.
    bool should_stop_checked(size_t s, int *rc) {
        for (;;) {
            std::vector<Item> items;
            bool winner_round = false;
            {
                std::lock_guard<std::mutex> lk(mu_);
                if (decided_ || shards_[s]->sc.saturated()) return true;
                if (!round_busy_) {
                    uint32_t nonce;
                    std::vector<uint64_t> idx;
                    const Plan p = plan_winner(0, &items, &nonce, &idx);   // the pass's lowest window decides the stop
                    if (p == DECIDED) { decided_ = true; return true; }
                    winner_round = round_busy_ = p == RECHECK;
                }
                if (!winner_round && !plan_saturation(s, &items)) return false;
            }
            *rc = round(shards_[s]->sc.engine(), items);
            if (winner_round) { std::lock_guard<std::mutex> lk(mu_); round_busy_ = false; }
            if (*rc) return true;
        }
    }

    bool checked_ = false, decided_ = false, round_busy_ = false;   // the last two under mu_
    uint8_t commitment_[32] = {0};
    uint64_t N_ = 0;
    const volatile int *cancel_ = nullptr;
    uint64_t rechecked_ = 0;                 // under mu_
    uint32_t rounds_ = 0;
    std::set<uint64_t> damaged_;
    int run_shard(size_t s, const Fill &fill, uint64_t chunk, uint64_t base, const volatile int *cancel) {
        Shard &sh = *shards_[s];
        Scanner &sc = sh.sc;
        std::mutex *mu = shards_.size() > 1 || checked_ ? &mu_ : nullptr;
        int rc = B200POST_OK;
        if (sh.lo == sh.hi) return rc;
        if (cudaSetDevice(sc.device()) != cudaSuccess) { cudaGetLastError(); set_error("cudaSetDevice failed"); return B200POST_ERR_CUDA; }
        int b = 0;
        for (uint64_t pos = sh.lo; pos < sh.hi; b ^= 1) {
            if (cancel && *cancel) { sc.drain(); set_error("cancelled"); return B200POST_ERR_CANCELLED; }
            if (abort_) { sc.drain(); return B200POST_OK; }   // another shard failed: its status is the call's
            if ((rc = sc.collect(b, mu))) { sc.drain(); return rc; }
            const bool stop = checked_ ? should_stop_checked(s, &rc) : should_stop(s);
            if (rc) { sc.drain(); return rc; }
            if (stop) break;
            // fill the staging buffer (a chunk may span files)
            const uint64_t n = std::min<uint64_t>(chunk, sh.hi - pos);
            if ((rc = fill(s, pos, n, sc.staging(b))) || (rc = sc.submit(b, base + pos, (uint32_t)n))) { sc.drain(); return rc; }
            pos += n;
        }
        for (int k = 0; k < 2; k++) if ((rc = sc.collect(b ^ k, mu))) { sc.drain(); return rc; }   // older chunk first
        return B200POST_OK;
    }

    // The unchecked stop rule, over the nonces of the pass's lowest window (a saturated shard has every nonce of the
    // pass at K2, that window's included)
    bool should_stop(size_t s) {
        if (shards_.size() == 1) {
            if (windows_ == 1) return shards_[0]->sc.any_full();
            const HitLists &l = shards_[0]->sc.lists();
            for (auto kv = l.lower_bound(first_); kv != l.end() && kv->first < first_ + window_; ++kv)
                if (kv->second.size() >= k2_) return true;
            return false;
        }
        std::lock_guard<std::mutex> lk(mu_);
        if (shards_[s]->sc.saturated()) return true;
        below_x_.assign(window_, 0);   // hits below x per nonce of the window
        for (const auto &sh : shards_) {
            const HitLists &l = sh->sc.lists();
            for (auto kv = l.lower_bound(first_); kv != l.end() && kv->first < first_ + window_; ++kv)
                if ((below_x_[kv->first - first_] += kv->second.size()) >= k2_) return true;
            if (sh->sc.scanned() < sh->hi - sh->lo && !sh->sc.saturated()) break;   // x lies in this shard
        }
        return false;
    }

    uint32_t first_, window_, windows_, k2_;
    std::vector<std::unique_ptr<Shard>> shards_;
    std::mutex mu_;                  // guards every shard's hit lists and progress once the threads run
    std::vector<uint64_t> below_x_;
    std::atomic<bool> abort_{false};
};

}  // namespace

int write_proof(uint64_t scanned, uint32_t nonce, const std::vector<uint64_t> &idx, const uint64_t *pows, uint32_t first_nonce,
                uint64_t num_labels, b200post_proof_out *out) {
    metrics().prove_labels_scanned_total += scanned; metrics().proofs_generated_total++;
    memset(out, 0, sizeof *out);
    out->nonce = nonce; out->pow = pows[(nonce - first_nonce) / 16]; out->labels_scanned = scanned;
    out->indices_len = b200post_pack_indices(idx.data(), idx.size(), b200post_bits_per_index(num_labels), out->indices, sizeof out->indices);
    if (out->indices_len == 0) { set_error("packed indices exceed the 800-byte wire cap"); return B200POST_ERR_INVALID_ARGUMENT; }
    return B200POST_OK;
}

const char *const kNoProof = "no proof found: no nonce reached K2 qualifying labels";

int check_pow_mode(const b200post_prove_opts &o) {
    if (o.pow_mode > B200POST_POW_SKIP || (o.pow_mode == B200POST_POW_CALLBACK && !o.pow_prove)) {
        set_error("pow_mode CALLBACK needs a pow_prove function; to prove without k2pow ask for B200POST_POW_SKIP explicitly");
        return B200POST_ERR_UNSUPPORTED;
    }
    return B200POST_OK;
}

int find_pows(const b200post_prove_opts &o, const uint8_t challenge[32], const uint8_t node_id[32], uint32_t num_units,
              const uint8_t cfg_difficulty[32], const uint32_t *providers, int n_providers, uint32_t first_group, uint32_t n_groups,
              std::vector<uint64_t> *pows, const volatile int *cancel) {
    pows->assign(n_groups, 0);
    if (o.pow_mode == B200POST_POW_SKIP) return B200POST_OK;
    uint8_t scaled[32];
    div256_u32(cfg_difficulty, num_units, scaled);
    if (o.pow_mode == B200POST_POW_CALLBACK) {
        for (uint32_t g = 0; g < n_groups; g++)
            if (o.pow_prove(o.pow_ctx, (uint8_t)(first_group + g), challenge, scaled, node_id, &(*pows)[g]) != 0) {
                set_error("k2pow hook failed");
                return B200POST_ERR_INVALID_ARGUMENT;
            }
        return B200POST_OK;
    }
    // the k2pow step of NIPostBuilder.Proof (activation/nipost.go:171 -> post-service): RandomX nonce search on the device
    b200post_k2pow_params kp{};
    kp.cache_key = o.pow_cache_key; kp.cache_key_len = o.pow_cache_key_len;
    memcpy(kp.challenge8, challenge, 8);
    memcpy(kp.node_id, node_id, 32);
    memcpy(kp.difficulty, scaled, 32);
    const int rc = b200post_k2pow_search_group_range_multi(providers, n_providers, &kp, first_group, n_groups, 0, pows->data(), nullptr, cancel);
    if (rc) return rc;
    for (uint64_t v : *pows) if (v == B200POST_K2POW_NOT_FOUND) { set_error("k2pow: nonce space exhausted"); return B200POST_ERR_INVALID_PROOF; }
    return B200POST_OK;
}

int gate_proof(uint32_t provider, const b200post_post_config &cfg, uint64_t scrypt_n, const b200post_prove_opts &o,
               const b200post_proof_metadata &meta, b200post_proof_out *out) {
    b200post_verify_params vp{};
    vp.k1 = cfg.k1; vp.k2 = cfg.k2; vp.scrypt_n = scrypt_n;
    memcpy(vp.pow_difficulty, cfg.pow_difficulty, 32);
    b200post_verifier_opts vo{};
    vo.pow_mode = o.pow_mode == B200POST_POW_BUILTIN ? B200POST_POW_BUILTIN : B200POST_POW_SKIP;
    vo.pow_cache_key = o.pow_cache_key; vo.pow_cache_key_len = o.pow_cache_key_len;
    const b200post_proof proof{out->nonce, out->indices, out->indices_len, out->pow};
    int status = B200POST_OK;
    uint64_t bad = 0;
    const int rc = b200post_verify_batch(provider, 1, &proof, &meta, &vp, nullptr, &vo, &status, &bad);
    if (rc) return rc;
    if (status != B200POST_OK) {
        memset(out, 0, sizeof *out);
        set_error(bad == ~0ull ? "the proof failed the verifier's k2pow check" : "the proof failed the verifier at position " + std::to_string(bad));
        return B200POST_ERR_INVALID_PROOF;
    }
    return B200POST_OK;
}

namespace {

// The checked proof's decision step for one pass: recheck rounds until the winner over usable hits is known (false: the
// pass has none), then the report, which adds up over the passes (`damaged`: every distinct damaged index so far).
bool decide_checked(ShardedScan &scan, uint32_t *nonce, std::vector<uint64_t> *idx, std::set<uint64_t> *damaged,
                    b200post_prove_check *check, int *rc) {
    const bool have = scan.decide(nonce, idx, rc);
    const size_t before = damaged->size();
    damaged->insert(scan.damaged().begin(), scan.damaged().end());
    check->labels_rechecked += scan.rechecked(); check->rounds += scan.rounds(); check->damaged = damaged->size();
    check->n_reported = 0;
    for (uint64_t i : *damaged) {   // ascending
        if (check->n_reported == 64) break;
        check->damaged_index[check->n_reported++] = i;
    }
    metrics().prove_labels_rechecked_total += scan.rechecked();
    metrics().prove_damaged_labels_total += damaged->size() - before;
    return have;
}

}  // namespace
}  // namespace b200post

using namespace b200post;

namespace {
// the same for labels already in (pageable) host memory
void parallel_copy(uint8_t *dst, const uint8_t *src, size_t bytes) {
    const size_t kMinSlice = (size_t)4 << 20;
    const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    const size_t nt = std::min<size_t>({(size_t)8, (size_t)hw, std::max<size_t>(1, bytes / kMinSlice)});
    if (nt <= 1) { memcpy(dst, src, bytes); return; }
    std::vector<std::thread> th;
    const size_t per = (bytes / nt + 63) & ~(size_t)63;
    for (size_t t = 0; t < nt; t++) {
        const size_t lo = std::min(bytes, t * per), hi = t + 1 == nt ? bytes : std::min(bytes, (t + 1) * per);
        th.emplace_back([=] { memcpy(dst + lo, src + lo, hi - lo); });
    }
    for (auto &x : th) x.join();
}
}  // namespace

namespace {
int generate(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg, const b200post_prove_opts *opts,
             const uint32_t *providers, int n_providers, b200post_proof_out *out, b200post_proof_metadata *meta_out,
             b200post_prove_check *check, const volatile int *cancel);
}  // namespace

extern "C" {

int b200post_prove_scan(uint32_t provider, const uint8_t *labels16, uint64_t first_index, uint64_t count, const uint8_t challenge[32],
                        uint32_t nonces, const uint64_t *pows, uint32_t k1, uint32_t k2, uint64_t num_labels, b200post_proof_out *out) {
    if (!labels16 || !challenge || !pows || !out) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    ShardedScan scan(1, 0, nonces, 1, k2);
    Shard &sh = scan.shard(0);
    const uint64_t chunk = std::min<uint64_t>(std::max<uint64_t>(count, 1), 1u << 22);
    int rc = sh.sc.init(provider, challenge, nonces, pows, k1, k2, num_labels, chunk);
    if (rc) return rc;
    sh.lo = 0; sh.hi = count;
    rc = scan.run([&](size_t, uint64_t off, uint64_t n, uint8_t *dst) {
        parallel_copy(dst, labels16 + off * 16, (size_t)n * 16);   // pageable -> pinned staging, the scan's host-side bound
        return B200POST_OK;
    }, chunk, first_index, nullptr);
    if (rc) return rc;
    uint32_t nonce = 0;
    std::vector<uint64_t> idx;
    if (!scan.winner(&nonce, &idx)) { set_error(kNoProof); return B200POST_ERR_INVALID_PROOF; }
    return write_proof(scan.scanned(), nonce, idx, pows, 0, num_labels, out);
}

int b200post_generate_proof(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg,
                            const b200post_prove_opts *opts, b200post_proof_out *out, b200post_proof_metadata *meta_out,
                            const volatile int *cancel) {
    const uint32_t provider = opts ? opts->provider : 0;
    return b200post_generate_proof_multi(data_dir, challenge, cfg, opts, &provider, 1, out, meta_out, cancel);
}

int b200post_generate_proof_multi(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg,
                                  const b200post_prove_opts *opts, const uint32_t *providers, int n_providers,
                                  b200post_proof_out *out, b200post_proof_metadata *meta_out, const volatile int *cancel) {
    if (!data_dir || !challenge || !cfg || !out || !providers || n_providers <= 0) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    return generate(data_dir, challenge, cfg, opts, providers, n_providers, out, meta_out, nullptr, cancel);
}

int b200post_generate_proof_checked(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg,
                                    const b200post_prove_opts *opts, const uint32_t *providers, int n_providers,
                                    b200post_proof_out *out, b200post_proof_metadata *meta_out, b200post_prove_check *check,
                                    const volatile int *cancel) {
    if (!data_dir || !challenge || !cfg || !out || !providers || n_providers <= 0 || !check) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    memset(check, 0, sizeof *check);
    return generate(data_dir, challenge, cfg, opts, providers, n_providers, out, meta_out, check, cancel);
}

}  // extern "C"

namespace {
// b200post_generate_proof_multi (check == nullptr) and b200post_generate_proof_checked: they differ only in the scan's
// hit records and the decision step (ShardedScan::enable_check, finish_checked) and the final verifier gate
int generate(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg, const b200post_prove_opts *opts,
             const uint32_t *providers, int n_providers, b200post_proof_out *out, b200post_proof_metadata *meta_out,
             b200post_prove_check *check, const volatile int *cancel) {
    b200post_prove_opts o{};
    if (opts) o = *opts;
    if (o.nonces == 0) o.nonces = 16;
    if (o.chunk_labels == 0) o.chunk_labels = 1ull << 22;
    b200post_post_metadata md;
    int rc = b200post_load_metadata(data_dir, &md);
    if (rc) return rc;
    const uint64_t num_labels = (uint64_t)md.num_units * md.labels_per_unit;
    if (num_labels == 0 || o.nonces % 16 || o.nonces > 4096) { set_error("invalid metadata or nonce count"); return B200POST_ERR_INVALID_ARGUMENT; }
    if (check && (md.scrypt_n < 2 || md.scrypt_n > (1ull << 20) || (md.scrypt_n & (md.scrypt_n - 1)))) {
        set_error("corrupt metadata: Scrypt.N out of range");
        return B200POST_ERR_IO;
    }
    if ((rc = check_pow_mode(o))) return rc;
    // the nonce windows [w*n, (w+1)*n) to try, `per_pass` of them per read of the data (b200post_prove_opts)
    const uint32_t n = o.nonces, windows = std::min(std::max(o.max_windows, 1u), 4096 / n);
    const uint32_t per_pass = std::max(o.windows_per_pass, 1u);
    const uint64_t chunk = std::min<uint64_t>(o.chunk_labels, num_labels);
    const auto ranges = split_shards(num_labels, chunk, (size_t)n_providers);
    uint8_t commitment[32];
    if (check) commitment_bytes(md.node_id, md.commitment_atx_id, commitment);
    const uint64_t per_file = md.max_file_size / 16;
    uint64_t scanned = 0;              // over every pass
    std::set<uint64_t> damaged;        // the checked report's, over every pass
    bool have = false;
    for (uint32_t a = 0; a < windows && !have;) {
        const uint32_t m = std::min(per_pass, windows - a), first = a * n;
        // k2pow per nonce group of the pass (RandomX upstream; or the caller's hook)
        std::vector<uint64_t> pows;
        if ((rc = find_pows(o, challenge, md.node_id, md.num_units, cfg->pow_difficulty, providers, n_providers, first / 16, m * n / 16,
                            &pows, cancel)))
            return rc;
        // one shard per list entry: its own Scanner (device buffers, double-buffered staging), reader and host thread
        ShardedScan scan((size_t)n_providers, first, n, m, cfg->k2);
        if (check) scan.enable_check(commitment, md.scrypt_n, cancel);
        for (int s = 0; s < n_providers; s++) {
            Shard &sh = scan.shard((size_t)s);
            if ((rc = sh.sc.init(providers[s], challenge, m * n, pows.data(), cfg->k1, cfg->k2, num_labels, chunk, check != nullptr, first)))
                return rc;
            sh.lo = ranges[(size_t)s].first; sh.hi = ranges[(size_t)s].second;
        }
        if (per_file == 0) { set_error("corrupt metadata: MaxFileSize"); return B200POST_ERR_IO; }
        std::vector<std::unique_ptr<PostDataReader>> readers;
        for (int s = 0; s < n_providers; s++) readers.emplace_back(new PostDataReader(data_dir, per_file));
        rc = scan.run([&](size_t s, uint64_t pos, uint64_t cnt, uint8_t *dst) { return readers[s]->read(pos, cnt, dst); }, chunk, 0, cancel);
        if (rc) return rc;
        metrics().prove_passes_total++;
        scanned += scan.scanned();
        uint32_t nonce = 0;
        std::vector<uint64_t> idx;
        have = check ? decide_checked(scan, &nonce, &idx, &damaged, check, &rc) : scan.winner(&nonce, &idx);
        if (rc) return rc;
        if (have && (rc = write_proof(scanned, nonce, idx, pows.data(), first, num_labels, out))) return rc;
        a += m;
    }
    if (!have) {
        set_error(windows == 1 ? std::string(kNoProof)
                               : std::string(kNoProof) + " in nonce windows 0.." + std::to_string(windows - 1) + " (nonces [0, " +
                                     std::to_string((uint64_t)windows * n) + "))");
        return B200POST_ERR_INVALID_PROOF;
    }
    b200post_proof_metadata meta;
    memcpy(meta.node_id, md.node_id, 32);
    memcpy(meta.commitment_atx_id, md.commitment_atx_id, 32);
    memcpy(meta.challenge, challenge, 32);
    meta.num_units = md.num_units; meta.labels_per_unit = md.labels_per_unit;
    if (check) {
        // the gate: a proof this library's own verifier rejects is never handed out
        if ((rc = gate_proof(providers[0], *cfg, md.scrypt_n, o, meta, out))) return rc;
        check->proof_verified = 1;
    }
    if (meta_out) *meta_out = meta;
    return B200POST_OK;
}
}  // namespace
