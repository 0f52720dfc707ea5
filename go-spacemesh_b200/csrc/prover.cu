// prover.cu — POST proof generation scan (include/b200post_prove.h, SURVEY.md §8f.3).
//
// K6 prove_scan_kernel streams 16-byte labels (H2D from the postdata files, double-buffered) through one
// AES-128 cipher per nonce group and appends (nonce, index) hits to a small list; the host folds them into per-nonce
// hit books and stops, under the rule of prove_rule.h, once a nonce owns K2 of them.  Bandwidth view: 16 B in per
// label, ~nothing out; the kernel is far faster than PCIe/NVMe can feed it, so the design goal is simply to keep copies
// and compute overlapped.  Conventions: post-rs Prover8_56 from memory (ASSUMED, unpinned).
//
// Several devices (b200post_generate_proof_multi): the label range is split into contiguous shards, one host thread,
// Scanner and hit book each (ShardedScan); the rule reads the books in shard order, so the proof is the one-device proof.
//
// Damaged stored data (b200post_generate_proof_checked): the same rule, with hits born pending instead of good.  The
// kernels also return each hit's stored bytes (StoredHit), and the tentative winner has its first K2 hits recomputed and
// compared on the device before the scan may stop on it; damaged hits are dropped (DESIGN.md §5).
//
// Checksummed data (b200post_generate_proof_sums): the checked scan over a chunk plan of whole digest ranges
// (sums_plan.h).  Each chunk's covered ranges are hashed on the device after its H2D and compared with their sidecar at
// collect; a bad range is recomputed into the chunk's device buffer and scanned again, covered hits are folded good and
// only uncovered ones pending (DESIGN.md §5).
//
// Nonce windows (b200post_prove_opts.max_windows): generate() runs passes over the data, each scanning windows_per_pass
// windows of nonces with their own pows, until a window has a proof; the kernels only ever see pass-relative nonces.
//
// Several identities (b200post_generate_proofs): prove_items runs every identity's pass loop; the pows of all identities
// waiting for a pass come from one k2pow job search, and each identity's scan starts as soon as its pows are final.  The
// single calls are its one-item case.
//
// The scanner, the proof record, the pow step and the verifier gate are declared in prove_internal.h: the setup
// session's initial proof (initial_proof.cu) runs the same scan over the labels as it writes them.
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdio>
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
#include "randomx_engine.h"

namespace b200post {
namespace {

struct Hit { uint32_t nonce; uint32_t pad; uint64_t index; };
// b200post_generate_proof_checked's record: the hit and the 16 stored bytes the kernel judged
struct StoredHit { uint32_t nonce; uint32_t pad; uint64_t index; uint4 label; };

__device__ __forceinline__ Hit make_hit(const Hit *, uint32_t nonce, uint64_t index, uint4) { return Hit{nonce, 0, index}; }
__device__ __forceinline__ StoredHit make_hit(const StoredHit *, uint32_t nonce, uint64_t index, uint4 label) {
    return StoredHit{nonce, 0, index, label};
}
// what the host folds into the hit book as the hit's stored bytes
const uint8_t *stored_bytes(const Hit &) { return nullptr; }
const uint8_t *stored_bytes(const StoredHit &h) { return reinterpret_cast<const uint8_t *>(&h.label); }

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

int Scanner::init(uint32_t provider, const uint8_t challenge[32], uint32_t nonces, const uint64_t *pows, uint32_t k1, uint32_t k2,
                  uint64_t num_labels, uint64_t chunk, bool keep_stored, uint32_t first_nonce) {
    DeviceEngine *e;
    if (int rc = device_engine(provider, &e)) return rc;
    if (nonces == 0 || nonces % 16 || first_nonce % 16 || (uint64_t)first_nonce + nonces > 4096 || k1 == 0 || k2 == 0 ||
        num_labels == 0 || chunk == 0 || chunk > (1u << 28)) {
        set_error("invalid proving parameters (nonces must be a positive multiple of 16, <= 4096)");
        return B200POST_ERR_INVALID_ARGUMENT;
    }
    engine_ = e; dev_ = e->device(); nonces_ = nonces; first_ = first_nonce; chunk_ = chunk;
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
void Scanner::launch(cudaStream_t st, const uint4 *labels, uint64_t first, uint32_t count, Rec *hits, uint32_t *n_hits, uint2 *cands,
                     uint32_t cand_cap, uint32_t *n_cands) {
    prove_scan_kernel<Rec><<<grid_, 256, AES_SMEM_BYTES, st>>>(labels, first, count, reinterpret_cast<const uint4 *>(d_rk_.get()), nonces_ / 16,
                                                               msb_, d_tables_.get(), hits, hit_cap_, n_hits, cands, cand_cap, n_cands);
    prove_lazy_kernel<Rec><<<grid_, 256, AES_SMEM_BYTES, st>>>(labels, first, cands, n_cands, cand_cap,
                                                               reinterpret_cast<const uint4 *>(d_lazy_.get()), lsb_, d_tables_.get(),
                                                               hits, hit_cap_, n_hits);
}

int Scanner::use_sums(SumsCheck *sums, const uint8_t commitment[32], uint64_t N, size_t max_ranges, const volatile int *cancel) {
    if (!stored_) { set_error("a checksummed scan keeps its hits' stored bytes"); return B200POST_ERR_INVALID_ARGUMENT; }
    sums_ = sums; N_ = N; cancel_ = cancel;
    memcpy(commitment_, commitment, 32);
    CUDA_TRY(cudaSetDevice(dev_));
    const size_t n = std::max<size_t>(max_ranges, 1);
    for (int b = 0; b < 2; b++) {
        CUDA_TRY(h_desc_[b].resize(n));
        CUDA_TRY(d_desc_[b].resize(n));
        CUDA_TRY(h_dig_[b].resize(n * 32));
        CUDA_TRY(d_dig_[b].resize(n * 32));
        hashed_[b].reserve(n);
    }
    heal_cand_cap_ = (uint32_t)((kSumBlockLabels * nonces_) / 128 + 65536);
    CUDA_TRY(d_heal_hits_.resize((size_t)hit_cap_ * rec_));
    CUDA_TRY(h_heal_hits_.resize((size_t)hit_cap_ * rec_));
    CUDA_TRY(d_heal_cands_.resize(heal_cand_cap_));
    CUDA_TRY(d_heal_n_.resize(2));
    CUDA_TRY(h_heal_n_.resize(2));
    CUDA_TRY(d_heal_dig_.resize(32));
    CUDA_TRY(h_heal_dig_.resize(32));
    CUDA_TRY(d_heal_desc_.resize(1));
    CUDA_TRY(h_heal_desc_.resize(1));
    return B200POST_OK;
}

int Scanner::submit(int b, uint64_t first, uint32_t count, const SumRange *ranges, size_t n_ranges) {
    CUDA_TRY(cudaMemcpyAsync(d_labels_[b].get(), h_labels_[b].get(), (size_t)count * 16, cudaMemcpyHostToDevice, st_[b].get()));
    if (sums_) {   // the covered ranges' digests, from the bytes K6a/K6b are about to read
        first_label_[b] = first; ranges_[b] = ranges; n_ranges_[b] = n_ranges;
        hashed_[b].clear();
        for (size_t i = 0; i < n_ranges; i++)
            if (ranges[i].sum) {
                h_desc_[b].get()[hashed_[b].size()] = DigestDesc{(ranges[i].first - first) * 16, (uint32_t)(ranges[i].count * 16), 0};
                hashed_[b].push_back(i);
            }
        const uint32_t nh = (uint32_t)hashed_[b].size();
        if (nh) {
            CUDA_TRY(cudaMemcpyAsync(d_desc_[b].get(), h_desc_[b].get(), nh * sizeof(DigestDesc), cudaMemcpyHostToDevice, st_[b].get()));
            CUDA_TRY(launch_range_digests(st_[b].get(), d_labels_[b].get(), d_desc_[b].get(), nh, d_dig_[b].get()));
            CUDA_TRY(cudaMemcpyAsync(h_dig_[b].get(), d_dig_[b].get(), (size_t)nh * 32, cudaMemcpyDeviceToHost, st_[b].get()));
        }
    }
    CUDA_TRY(cudaMemsetAsync(d_nhits_[b].get(), 0, 4, st_[b].get()));
    // the single candidate queue is reused by consecutive chunks: wait for the other stream's lazy pass
    if (pending_[b ^ 1]) CUDA_TRY(cudaStreamWaitEvent(st_[b].get(), ev_[b ^ 1].get(), 0));
    CUDA_TRY(cudaMemsetAsync(d_ncands_.get(), 0, 8, st_[b].get()));
    cudaStream_t st = st_[b].get();
    const uint4 *labels = reinterpret_cast<const uint4 *>(d_labels_[b].get());
    if (stored_) launch(st, labels, first, count, reinterpret_cast<StoredHit *>(d_hits_[b].get()), d_nhits_[b].get(), d_cands_.get(), cand_cap_, d_ncands_.get());
    else launch(st, labels, first, count, reinterpret_cast<Hit *>(d_hits_[b].get()), d_nhits_[b].get(), d_cands_.get(), cand_cap_, d_ncands_.get());
    g_launches += 2;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(h_ncands_[b].get(), d_ncands_.get(), 4, cudaMemcpyDeviceToHost, st_[b].get()));
    CUDA_TRY(cudaMemcpyAsync(h_nhits_[b].get(), d_nhits_[b].get(), 4, cudaMemcpyDeviceToHost, st_[b].get()));
    CUDA_TRY(cudaMemcpyAsync(h_hits_[b].get(), d_hits_[b].get(), (size_t)hit_cap_ * rec_, cudaMemcpyDeviceToHost, st_[b].get()));
    CUDA_TRY(cudaEventRecord(ev_[b].get(), st_[b].get()));
    pending_[b] = true; count_[b] = count;
    return B200POST_OK;
}

int Scanner::collect(int b, HitBook *book, std::mutex *fold_mu) {
    if (!pending_[b]) return B200POST_OK;
    CUDA_TRY(cudaEventSynchronize(ev_[b].get()));
    pending_[b] = false;
    const uint32_t n = *h_nhits_[b].get();
    if (n > hit_cap_ || *h_ncands_[b].get() > cand_cap_) { set_error("hit buffer overflow: K1 too large for this chunk size"); return B200POST_ERR_OUT_OF_MEMORY; }
    if (sums_) return fold_sums(b, n, book, fold_mu);
    if (stored_) fold<StoredHit>(b, n, book, fold_mu);
    else fold<Hit>(b, n, book, fold_mu);
    return B200POST_OK;
}

template <class Rec>
void Scanner::fold(int b, uint32_t n, HitBook *book, std::mutex *fold_mu) {
    const Rec *rec = reinterpret_cast<const Rec *>(h_hits_[b].get());
    std::vector<Rec> v(rec, rec + n);
    std::sort(v.begin(), v.end(), [](const Rec &x, const Rec &y) { return x.index != y.index ? x.index < y.index : x.nonce < y.nonce; });
    std::unique_lock<std::mutex> lk;
    if (fold_mu) lk = std::unique_lock<std::mutex>(*fold_mu);
    for (const Rec &h : v) book->add(first_ + h.nonce, h.index, stored_bytes(h));
    book->advance(count_[b]);   // chunks are contiguous from the first index: the sum is how far the scan went
}

// One bad range of chunk b whose stored bytes hash to `stored`: its labels recomputed on this device's engine straight
// into the chunk's device buffer, then hashed (to classify the damage) and scanned into the heal buffers.  *hits: the
// range's StoredHit records.  Shards sharing a device serialise on its engine, as rechecks do.
int Scanner::heal(int b, const SumRange &r, const uint8_t stored[32], std::vector<uint8_t> *hits, bool *sidecar_only) {
    const uint64_t off = r.first - first_label_[b];
    uint8_t *dst = d_labels_[b].get() + off * 16;
    if (int rc = engine_->labels_range(commitment_, N_, r.first, r.count, nullptr, dst, nullptr, nullptr, cancel_)) return rc;
    CUDA_TRY(cudaSetDevice(dev_));
    cudaStream_t st = st_[b].get();
    *h_heal_desc_.get() = DigestDesc{off * 16, (uint32_t)(r.count * 16), 0};
    CUDA_TRY(cudaMemcpyAsync(d_heal_desc_.get(), h_heal_desc_.get(), sizeof(DigestDesc), cudaMemcpyHostToDevice, st));
    CUDA_TRY(launch_range_digests(st, d_labels_[b].get(), d_heal_desc_.get(), 1, d_heal_dig_.get()));
    CUDA_TRY(cudaMemsetAsync(d_heal_n_.get(), 0, 8, st));
    launch(st, reinterpret_cast<const uint4 *>(dst), r.first, (uint32_t)r.count, reinterpret_cast<StoredHit *>(d_heal_hits_.get()),
           d_heal_n_.get(), d_heal_cands_.get(), heal_cand_cap_, d_heal_n_.get() + 1);
    g_launches += 2;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(h_heal_dig_.get(), d_heal_dig_.get(), 32, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(h_heal_n_.get(), d_heal_n_.get(), 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    const uint32_t n = h_heal_n_.get()[0];
    if (n > hit_cap_ || h_heal_n_.get()[1] > heal_cand_cap_) { set_error("hit buffer overflow: K1 too large for this chunk size"); return B200POST_ERR_OUT_OF_MEMORY; }
    CUDA_TRY(cudaMemcpyAsync(h_heal_hits_.get(), d_heal_hits_.get(), (size_t)n * rec_, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    hits->assign(h_heal_hits_.get(), h_heal_hits_.get() + (size_t)n * rec_);
    // the stored bytes' digest equals the recomputation's: the data is right and the sidecar's digest is wrong
    *sidecar_only = memcmp(h_heal_dig_.get(), stored, 32) == 0;
    return B200POST_OK;
}

// collect of a checksummed chunk: the covered ranges' digests compared with their sidecar's, the bad ones counted
// against the heal cap and healed, then the fold.  A hit's state comes from its range: covered (the digest matched, or
// the range was recomputed) is good, uncovered is pending; a bad range's stored hits are replaced by its healed ones.
int Scanner::fold_sums(int b, uint32_t n, HitBook *book, std::mutex *fold_mu) {
    const SumRange *r = ranges_[b];
    const size_t nr = n_ranges_[b];
    std::vector<uint8_t> bad(nr, 0);
    std::vector<size_t> bad_list;
    uint64_t verified = 0, uncovered = 0;
    for (size_t k = 0; k < hashed_[b].size(); k++) {
        const size_t i = hashed_[b][k];
        if (memcmp(h_dig_[b].get() + k * 32, r[i].sum, 32) == 0) verified += r[i].count;
        else { bad[i] = 1; bad_list.push_back(k); }
    }
    for (size_t i = 0; i < nr; i++) if (!r[i].sum) uncovered += r[i].count;
    sums_->blocks_checked += hashed_[b].size();
    sums_->labels_verified += verified;
    sums_->labels_uncovered += uncovered;
    const StoredHit *rec = reinterpret_cast<const StoredHit *>(h_hits_[b].get());
    std::vector<StoredHit> v;
    v.reserve(n);
    const auto range_of = [&](uint64_t index) {   // the range holding a label of the chunk
        size_t lo = 0, hi = nr;
        while (hi - lo > 1) { const size_t m = (lo + hi) / 2; (r[m].first <= index ? lo : hi) = m; }
        return lo;
    };
    for (uint32_t j = 0; j < n; j++) if (!bad[range_of(rec[j].index)]) v.push_back(rec[j]);
    if (!bad_list.empty()) {
        {
            std::lock_guard<std::mutex> g(sums_->mu);
            for (size_t k : bad_list) {
                const SumRange &x = r[hashed_[b][k]];
                sums_->bad.emplace(x.first, SumsCheck::Bad{x.count, false});
            }
            if (sums_->bad.size() > sums_->max_heal) {
                set_error("more than " + std::to_string(sums_->max_heal) + " damaged blocks: repair first (b200postcli -checkSums -repair)");
                return B200POST_ERR_LABEL_MISMATCH;
            }
        }
        for (size_t k : bad_list) {
            const SumRange &x = r[hashed_[b][k]];
            std::vector<uint8_t> healed;
            bool sidecar_only = false;
            if (int rc = heal(b, x, h_dig_[b].get() + k * 32, &healed, &sidecar_only)) return rc;
            const StoredHit *h = reinterpret_cast<const StoredHit *>(healed.data());
            v.insert(v.end(), h, h + healed.size() / sizeof(StoredHit));
            std::lock_guard<std::mutex> g(sums_->mu);
            sums_->bad[x.first].sidecar_only = sidecar_only;
            sums_->healed.insert(x.first);
        }
    }
    std::sort(v.begin(), v.end(), [](const StoredHit &x, const StoredHit &y) { return x.index != y.index ? x.index < y.index : x.nonce < y.nonce; });
    std::unique_lock<std::mutex> lk;
    if (fold_mu) lk = std::unique_lock<std::mutex>(*fold_mu);
    for (const StoredHit &h : v) book->add(first_ + h.nonce, h.index, stored_bytes(h), r[range_of(h.index)].sum != nullptr);
    book->advance(count_[b]);
    return B200POST_OK;
}

void Scanner::drain() {
    for (int b = 0; b < 2; b++) if (pending_[b]) { cudaEventSynchronize(ev_[b].get()); pending_[b] = false; }
}

namespace {

// One contiguous label range [lo, hi) of a scan, streamed through its own Scanner.
struct Shard {
    Scanner sc;
    uint64_t lo = 0, hi = 0;
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

// One pass's scan split into shards, one host thread, Scanner and hit book each, driving the pass's ProveRule: its stop
// rule after every chunk, its decision once every thread has joined.  With a commitment (the checked proof) hits are
// born pending and the rule's recheck recomputes labels on the devices.
class ShardedScan {
public:
    // fill(shard, first label, count, dst): those labels into the shard's pinned staging
    using Fill = std::function<int(size_t, uint64_t, uint64_t, uint8_t *)>;

    // ranges[s]: shard s's labels [lo, hi); the pass scans `windows` nonce windows of `window` nonces from nonce `first`
    ShardedScan(const std::vector<std::pair<uint64_t, uint64_t>> &ranges, uint32_t first, uint32_t window, uint32_t windows,
                uint32_t k2, const uint8_t *commitment = nullptr, uint64_t N = 0, const volatile int *cancel = nullptr)
        : rule_(ranges, first, window, windows, k2, commitment ? ProveRule::Recheck([this](auto &&...a) { return recheck(a...); }) : nullptr),
          N_(N), cancel_(cancel) {
        if (commitment) memcpy(commitment_, commitment, 32);
        for (const auto &r : ranges) shards_.emplace_back(new Shard{{}, r.first, r.second});
    }
    Scanner &scanner(size_t s) { return shards_[s]->sc; }
    ProveRule &rule() { return rule_; }
    // the shards stream the plan's chunks (their ranges must be the plan's shards) instead of chunks of `chunk` labels
    void use_plan(const SumsPlan *plan) { plan_ = plan; }

    // runs every shard (the calling thread alone when there is one) and returns the first failing shard's status, in
    // list order, once every thread has joined
    int run(const Fill &fill, uint64_t chunk, uint64_t base, const volatile int *cancel) {
        if (shards_.size() == 1) return run_shard(0, fill, chunk, base, cancel);
        return fan_out(shards_.size(), [&](size_t s) {
            const int rc = run_shard(s, fill, chunk, base, cancel);
            if (rc != B200POST_OK) abort_ = true;
            return rc;
        });
    }

private:
    // The rule's recheck on shard s's device: the items' labels recomputed under the commitment and compared with their
    // stored bytes.  A compare reports at most CompareResult::kMaxReported positions, so it is repeated past the last
    // reported one until every mismatch is known.
    int recheck(size_t s, const std::vector<RecheckItem> &items, std::vector<uint8_t> *bad) {
        const size_t n = items.size();
        std::vector<uint64_t> idx(n);
        std::vector<uint8_t> expect(n * 16);
        for (size_t i = 0; i < n; i++) { idx[i] = items[i].index; memcpy(&expect[i * 16], items[i].label, 16); }
        for (size_t from = 0; from < n;) {
            CompareResult cmp;
            const int rc = shards_[s]->sc.engine()->labels_compare_indexed(commitment_, n - from, idx.data() + from, N_,
                                                                           expect.data() + from * 16, &cmp, cancel_);
            if (rc) return rc;
            for (uint64_t p : cmp.first) (*bad)[from + p] = 1;
            if (cmp.mismatches <= cmp.first.size()) break;
            from += cmp.first.back() + 1;
        }
        return B200POST_OK;
    }

    int run_shard(size_t s, const Fill &fill, uint64_t chunk, uint64_t base, const volatile int *cancel) {
        Shard &sh = *shards_[s];
        Scanner &sc = sh.sc;
        HitBook &book = rule_.book(s);
        int rc = B200POST_OK;
        if (sh.lo == sh.hi) return rc;
        if (cudaSetDevice(sc.device()) != cudaSuccess) { cudaGetLastError(); set_error("cudaSetDevice failed"); return B200POST_ERR_CUDA; }
        int b = 0;
        size_t k = plan_ ? plan_->shards[s].first : 0;   // the plan's next chunk
        for (uint64_t pos = sh.lo; pos < sh.hi; b ^= 1) {
            if (cancel && *cancel) { sc.drain(); set_error("cancelled"); return B200POST_ERR_CANCELLED; }
            if (abort_) { sc.drain(); return B200POST_OK; }   // another shard failed: its status is the call's
            if ((rc = sc.collect(b, &book, &mu_))) { sc.drain(); return rc; }
            const bool stop = rule_.should_stop(s, mu_, &rc);
            if (rc) { sc.drain(); return rc; }
            if (stop) break;
            // fill the staging buffer (a chunk may span files)
            const SumChunk *c = plan_ ? &plan_->chunks[k++] : nullptr;
            const uint64_t n = c ? c->count : std::min<uint64_t>(chunk, sh.hi - pos);
            if ((rc = fill(s, pos, n, sc.staging(b))) ||
                (rc = sc.submit(b, base + pos, (uint32_t)n, c ? &plan_->ranges[c->r0] : nullptr, c ? c->r1 - c->r0 : 0))) {
                sc.drain();
                return rc;
            }
            pos += n;
        }
        for (int k = 0; k < 2; k++) if ((rc = sc.collect(b ^ k, &book, &mu_))) { sc.drain(); return rc; }   // older chunk first
        return B200POST_OK;
    }

    ProveRule rule_;
    const SumsPlan *plan_ = nullptr;
    uint8_t commitment_[32] = {0};
    uint64_t N_ = 0;
    const volatile int *cancel_ = nullptr;
    std::vector<std::unique_ptr<Shard>> shards_;
    std::mutex mu_;                  // guards every shard's hit book and the rule's state once the threads run
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

int no_proof(uint32_t windows, uint32_t n) {
    std::string e = "no proof found: no nonce reached K2 qualifying labels";
    if (windows > 1) e += " in nonce windows 0.." + std::to_string(windows - 1) + " (nonces [0, " + std::to_string((uint64_t)windows * n) + "))";
    set_error(e);
    return B200POST_ERR_INVALID_PROOF;
}

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

void gate_proofs(uint32_t provider, const b200post_post_config &cfg, uint64_t scrypt_n, const b200post_prove_opts &o, size_t n,
                 const b200post_proof_metadata *metas, b200post_proof_out *const *outs, int *rcs, std::string *errs) {
    b200post_verify_params vp{};
    vp.k1 = cfg.k1; vp.k2 = cfg.k2; vp.scrypt_n = scrypt_n;
    memcpy(vp.pow_difficulty, cfg.pow_difficulty, 32);
    b200post_verifier_opts vo{};
    vo.pow_mode = o.pow_mode == B200POST_POW_BUILTIN ? B200POST_POW_BUILTIN : B200POST_POW_SKIP;
    vo.pow_cache_key = o.pow_cache_key; vo.pow_cache_key_len = o.pow_cache_key_len;
    std::vector<b200post_proof> proofs(n);
    for (size_t i = 0; i < n; i++) proofs[i] = b200post_proof{outs[i]->nonce, outs[i]->indices, outs[i]->indices_len, outs[i]->pow};
    std::vector<int> status(n, B200POST_OK);
    std::vector<uint64_t> bad(n, 0);
    const int rc = b200post_verify_batch(provider, n, proofs.data(), metas, &vp, nullptr, &vo, status.data(), bad.data());
    for (size_t i = 0; i < n; i++) {
        rcs[i] = rc ? rc : status[i] != B200POST_OK ? B200POST_ERR_INVALID_PROOF : B200POST_OK;
        if (rc) errs[i] = last_error();
        else if (status[i] != B200POST_OK) {
            memset(outs[i], 0, sizeof *outs[i]);
            errs[i] = bad[i] == ~0ull ? "the proof failed the verifier's k2pow check" : "the proof failed the verifier at position " + std::to_string(bad[i]);
        }
    }
}

int gate_proof(uint32_t provider, const b200post_post_config &cfg, uint64_t scrypt_n, const b200post_prove_opts &o,
               const b200post_proof_metadata &meta, b200post_proof_out *out) {
    int rc = B200POST_OK;
    std::string err;
    gate_proofs(provider, cfg, scrypt_n, o, 1, &meta, &out, &rc, &err);
    if (rc) set_error(err);
    return rc;
}

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

// One identity's proof in progress: its host checks' results and what the pass loop keeps between passes.  out, meta_out
// and check are the caller's (check is set for a checked proof).
struct ItemProof {
    const char *data_dir = nullptr;
    const uint8_t *challenge = nullptr;
    b200post_proof_out *out = nullptr;
    b200post_proof_metadata *meta_out = nullptr;
    b200post_prove_check *check = nullptr;
    SumsCheck *sums = nullptr;         // set for a checksummed proof (with check)
    b200post_post_metadata md{};
    uint64_t num_labels = 0, per_file = 0, chunk = 0;
    uint32_t n = 0, windows = 0, per_pass = 0;
    std::vector<std::pair<uint64_t, uint64_t>> ranges;
    std::vector<PostSums> sidecars;    // checksummed: per file, its usable sidecar (covering nothing without one)
    SumsPlan plan;                     // checksummed: the chunks and shards over the sidecars' digest ranges
    uint8_t commitment[32] = {0};
    uint32_t a = 0;                    // the next pass starts at window a
    uint64_t scanned = 0;              // over every pass
    std::set<uint64_t> damaged;        // the checked report's, over every pass
    bool have = false;
    std::vector<uint64_t> pows;        // the current pass's, one per nonce group
    b200post_proof_metadata meta{};
    int status = B200POST_OK;          // the single call's code and text once `done`
    std::string error;
    bool done = false;

    uint32_t pass_windows() const { return std::min(per_pass, windows - a); }
    uint32_t first_group() const { return a * n / 16; }
    uint32_t groups() const { return pass_windows() * n / 16; }
    void finish(int rc, const std::string &err) { status = rc; error = rc ? err : std::string(); done = true; }
};

// The host checks of one proof, in the single call's order: metadata, nonce count, scrypt N (checked), pow mode,
// MaxFileSize.  Then the pass plan.
int open_item(ItemProof &it, const b200post_prove_opts &o, int n_providers) {
    int rc = b200post_load_metadata(it.data_dir, &it.md);
    if (rc) return rc;
    const b200post_post_metadata &md = it.md;
    it.num_labels = (uint64_t)md.num_units * md.labels_per_unit;
    if (it.num_labels == 0 || o.nonces % 16 || o.nonces > 4096) { set_error("invalid metadata or nonce count"); return B200POST_ERR_INVALID_ARGUMENT; }
    if (it.check && (md.scrypt_n < 2 || md.scrypt_n > (1ull << 20) || (md.scrypt_n & (md.scrypt_n - 1)))) {
        set_error("corrupt metadata: Scrypt.N out of range");
        return B200POST_ERR_IO;
    }
    if ((rc = check_pow_mode(o))) return rc;
    it.per_file = md.max_file_size / 16;
    if (it.per_file == 0) { set_error("corrupt metadata: MaxFileSize"); return B200POST_ERR_IO; }
    // the nonce windows [w*n, (w+1)*n) to try, `per_pass` of them per read of the data (b200post_prove_opts)
    it.n = o.nonces;
    it.windows = std::min(std::max(o.max_windows, 1u), 4096 / it.n);
    it.per_pass = std::max(o.windows_per_pass, 1u);
    it.chunk = std::min<uint64_t>(o.chunk_labels, it.num_labels);
    it.ranges = split_shards(it.num_labels, it.chunk, (size_t)n_providers);
    if (it.check) commitment_bytes(md.node_id, md.commitment_atx_id, it.commitment);
    if (it.sums) {   // a missing or unusable sidecar only leaves its file uncovered
        const Layout lay(md);
        std::vector<SumsFile> files;
        it.sidecars.resize(lay.n_files);
        for (uint64_t f = 0; f < lay.n_files; f++) {
            PostSums &ps = it.sidecars[f];
            if (!load_post_sums(it.data_dir, md, f, lay.labels_in(f), &ps)) ps = PostSums::of(md, f);
            files.push_back({lay.labels_in(f), ps.covered, reinterpret_cast<const uint8_t *>(ps.digests.data())});
        }
        it.plan = plan_sums(files, o.chunk_labels, (size_t)n_providers);
        it.chunk = it.plan.max_chunk;
        for (size_t s = 0; s < it.ranges.size(); s++) it.ranges[s] = it.plan.shard_labels(s);
    }
    return B200POST_OK;
}

// One pass of an item with its pows found: the scan of windows [a, a + m), its rule's decision and the checked report.
// Marks the item done when it has a proof (before the gate) or no window is left.
int scan_pass(ItemProof &it, const b200post_post_config &cfg, const uint32_t *providers, int n_providers, const volatile int *cancel) {
    const uint32_t m = it.pass_windows(), first = it.a * it.n;
    // one shard per list entry: its own Scanner (device buffers, double-buffered staging), reader and host thread
    ShardedScan scan(it.ranges, first, it.n, m, cfg.k2, it.check ? it.commitment : nullptr, it.md.scrypt_n, cancel);
    if (it.sums) scan.use_plan(&it.plan);
    int rc;
    for (int s = 0; s < n_providers; s++) {
        Scanner &sc = scan.scanner((size_t)s);
        if ((rc = sc.init(providers[s], it.challenge, m * it.n, it.pows.data(), cfg.k1, cfg.k2, it.num_labels, it.chunk, it.check != nullptr, first)))
            return rc;
        if (it.sums && (rc = sc.use_sums(it.sums, it.commitment, it.md.scrypt_n, it.plan.max_ranges, cancel))) return rc;
    }
    std::vector<std::unique_ptr<PostDataReader>> readers;
    for (int s = 0; s < n_providers; s++) readers.emplace_back(new PostDataReader(it.data_dir, it.per_file));
    rc = scan.run([&](size_t s, uint64_t pos, uint64_t cnt, uint8_t *dst) { return readers[s]->read(pos, cnt, dst); }, it.chunk, 0, cancel);
    if (rc) return rc;
    metrics().prove_passes_total++;
    ProveRule &rule = scan.rule();
    it.scanned += rule.scanned();
    uint32_t nonce = 0;
    std::vector<uint64_t> idx;
    it.have = rule.decide(&nonce, &idx, &rc);
    if (b200post_prove_check *check = it.check) {   // the report adds up over the passes (`damaged`: every distinct damaged index so far)
        const size_t before = it.damaged.size();
        it.damaged.insert(rule.damaged().begin(), rule.damaged().end());
        check->labels_rechecked += rule.rechecked(); check->rounds += rule.rounds(); check->damaged = it.damaged.size();
        check->n_reported = 0;
        for (uint64_t i : it.damaged) {   // ascending
            if (check->n_reported == 64) break;
            check->damaged_index[check->n_reported++] = i;
        }
        metrics().prove_labels_rechecked_total += rule.rechecked();
        metrics().prove_damaged_labels_total += it.damaged.size() - before;
    }
    if (rc) return rc;
    if (it.have && (rc = write_proof(it.scanned, nonce, idx, it.pows.data(), first, it.num_labels, it.out))) return rc;
    it.a += m;
    if (!it.have && it.a < it.windows) return B200POST_OK;   // another pass
    if (!it.have) return no_proof(it.windows, it.n);
    memcpy(it.meta.node_id, it.md.node_id, 32);
    memcpy(it.meta.commitment_atx_id, it.md.commitment_atx_id, 32);
    memcpy(it.meta.challenge, it.challenge, 32);
    it.meta.num_units = it.md.num_units; it.meta.labels_per_unit = it.md.labels_per_unit;
    it.done = true;
    return B200POST_OK;
}

// The pass loop of every item (b200post_generate_proofs; the single calls are its one-item case).  The pows of every
// item waiting for a pass go into one search (BUILTIN: one k2pow job search over the devices; CALLBACK / SKIP: per item
// on this thread).  An item's scan starts on one of the scan threads as soon as its pows are final, while the search
// goes on for the others, and an item that needs another pass joins the next search.  Checked proofs then pass the
// verifier gate together.  Each item ends with its single call's status and text; the return value is the call's own:
// UNSUPPORTED for the pow mode, NO_DEVICE / UNSUPPORTED of the device list, CANCELLED, else OK.
int prove_items(std::vector<ItemProof> &items, const b200post_post_config &cfg, const b200post_prove_opts &o, const uint32_t *providers,
                int n_providers, uint32_t parallel_scans, const volatile int *cancel) {
    for (ItemProof &it : items)
        if (int rc = open_item(it, o, n_providers)) it.finish(rc, last_error());
    if (int rc = check_pow_mode(o)) return rc;   // every item that got this far answers the same
    std::mutex mu;                               // guards everything below and every item's done / status
    std::condition_variable cv;
    std::vector<size_t> waiting, ready;          // items needing the pows of their next pass; items to scan
    size_t left = 0;                             // items not done
    for (size_t i = 0; i < items.size(); i++) if (!items[i].done) { waiting.push_back(i); left++; }
    const auto end_item = [&](size_t i, int rc, const std::string &err) {   // under mu
        items[i].finish(rc, err);
        left--;
        cv.notify_all();
    };
    const auto scan_loop = [&] {
        std::unique_lock<std::mutex> lk(mu);
        for (;;) {
            cv.wait(lk, [&] { return !ready.empty() || left == 0; });
            if (ready.empty()) return;
            const size_t i = ready.front();
            ready.erase(ready.begin());
            lk.unlock();
            const int rc = scan_pass(items[i], cfg, providers, n_providers, cancel);
            const std::string err = rc ? last_error() : std::string();
            lk.lock();
            if (rc || items[i].done) end_item(i, rc, err);
            else { waiting.push_back(i); cv.notify_all(); }
        }
    };
    std::vector<std::thread> scanners;
    int call_rc = B200POST_OK;
    bool devices_checked = false;
    std::unique_lock<std::mutex> lk(mu);
    while (left) {
        cv.wait(lk, [&] { return !waiting.empty() || left == 0; });
        if (!left) break;
        std::vector<size_t> batch;
        batch.swap(waiting);
        std::sort(batch.begin(), batch.end());
        lk.unlock();
        std::vector<int> rcs(batch.size(), B200POST_OK);
        std::vector<std::string> errs(batch.size());
        std::vector<bool> handed(batch.size(), false);   // pows final: the item went to `ready`
        // the single call's pow step for the items without BUILTIN: their hooks, before any device is touched
        if (o.pow_mode != B200POST_POW_BUILTIN)
            for (size_t b = 0; b < batch.size(); b++) {
                ItemProof &it = items[batch[b]];
                if ((rcs[b] = find_pows(o, it.challenge, it.md.node_id, it.md.num_units, cfg.pow_difficulty, providers, n_providers,
                                        it.first_group(), it.groups(), &it.pows, cancel)))
                    errs[b] = last_error();
            }
        // the devices answer once, where the single call first touches them: the search (BUILTIN) or the first scan
        int rc = B200POST_OK;
        std::vector<RandomxEngine *> eng;
        if (!devices_checked) {
            devices_checked = true;
            if (o.pow_mode == B200POST_POW_BUILTIN) rc = randomx_engines(providers, n_providers, &eng);
            if (!rc) rc = device_engines(providers, n_providers);
            if (rc) call_rc = rc;
            else for (size_t t = std::min<size_t>(left, parallel_scans ? parallel_scans : 4); t; t--) scanners.emplace_back(scan_loop);
        }
        if (!rc && o.pow_mode == B200POST_POW_BUILTIN) {
            // one job search over the pass's nonce groups of every item in the batch
            std::vector<K2powJob> jobs;
            std::vector<size_t> owner, first_job(batch.size()), unfinal(batch.size());
            for (size_t b = 0; b < batch.size(); b++) {
                ItemProof &it = items[batch[b]];
                uint8_t scaled[32];
                div256_u32(cfg.pow_difficulty, it.md.num_units, scaled);
                first_job[b] = jobs.size();
                unfinal[b] = it.groups();
                it.pows.assign(it.groups(), B200POST_K2POW_NOT_FOUND);
                for (uint32_t g = 0; g < it.groups(); g++) {
                    K2powJob j;
                    j.tail[0] = (uint8_t)(it.first_group() + g);
                    memcpy(j.tail + 1, it.challenge, 8);
                    memcpy(j.tail + 9, it.md.node_id, 32);
                    memcpy(j.difficulty, scaled, 32);
                    jobs.push_back(j);
                    owner.push_back(b);
                }
            }
            if (eng.empty()) randomx_engines(providers, n_providers, &eng);
            const std::string key = o.pow_cache_key ? std::string(reinterpret_cast<const char *>(o.pow_cache_key), o.pow_cache_key_len)
                                                    : std::string(B200POST_K2POW_DEFAULT_KEY);
            std::vector<uint64_t> pows(jobs.size());
            rc = k2pow_search_jobs(eng, key, jobs, 0, pows.data(), nullptr, cancel, [&](uint32_t j, uint64_t pow) {
                const size_t b = owner[j];
                ItemProof &it = items[batch[b]];
                it.pows[j - first_job[b]] = pow;
                if (--unfinal[b]) return;
                std::lock_guard<std::mutex> g(mu);
                handed[b] = true;
                if (std::find(it.pows.begin(), it.pows.end(), B200POST_K2POW_NOT_FOUND) != it.pows.end()) {
                    end_item(batch[b], B200POST_ERR_INVALID_PROOF, "k2pow: nonce space exhausted");
                    return;
                }
                ready.push_back(batch[b]);
                cv.notify_all();
            });
        }
        const std::string err = rc ? last_error() : std::string();
        lk.lock();
        for (size_t b = 0; b < batch.size(); b++) {
            if (handed[b]) continue;
            if (rcs[b]) end_item(batch[b], rcs[b], errs[b]);       // its hook failed
            else if (rc) end_item(batch[b], rc, err);              // the devices or the search failed before its pows were final
            else { ready.push_back(batch[b]); cv.notify_all(); }   // CALLBACK / SKIP pows
        }
    }
    lk.unlock();
    for (std::thread &t : scanners) t.join();
    // the gate: the checked proofs of each scrypt N in one b200post_verify_batch call on the first device
    std::map<uint64_t, std::vector<size_t>> gate;
    for (size_t i = 0; i < items.size(); i++)
        if (items[i].status == B200POST_OK && items[i].check) gate[items[i].md.scrypt_n].push_back(i);
    for (const auto &kv : gate) {
        const size_t k = kv.second.size();
        std::vector<b200post_proof_metadata> metas(k);
        std::vector<b200post_proof_out *> outs(k);
        std::vector<int> rcs(k);
        std::vector<std::string> errs(k);
        for (size_t g = 0; g < k; g++) { metas[g] = items[kv.second[g]].meta; outs[g] = items[kv.second[g]].out; }
        gate_proofs(providers[0], cfg, kv.first, o, k, metas.data(), outs.data(), rcs.data(), errs.data());
        for (size_t g = 0; g < k; g++) {
            ItemProof &it = items[kv.second[g]];
            if (rcs[g]) it.finish(rcs[g], errs[g]);
            else it.check->proof_verified = 1;
        }
    }
    for (ItemProof &it : items) {
        if (it.status == B200POST_OK && it.meta_out) *it.meta_out = it.meta;
        if (it.status == B200POST_ERR_CANCELLED && !call_rc) call_rc = B200POST_ERR_CANCELLED;
    }
    if (call_rc == B200POST_ERR_CANCELLED) set_error("cancelled");
    return call_rc;
}

int generate(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg, const b200post_prove_opts *opts,
             const uint32_t *providers, int n_providers, b200post_proof_out *out, b200post_proof_metadata *meta_out,
             b200post_prove_check *check, const volatile int *cancel, SumsCheck *sums = nullptr);
b200post_prove_opts prove_opts(const b200post_prove_opts *opts);

}  // namespace

extern "C" {

int b200post_prove_scan(uint32_t provider, const uint8_t *labels16, uint64_t first_index, uint64_t count, const uint8_t challenge[32],
                        uint32_t nonces, const uint64_t *pows, uint32_t k1, uint32_t k2, uint64_t num_labels, b200post_proof_out *out) {
    if (!labels16 || !challenge || !pows || !out) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    ShardedScan scan({{0, count}}, 0, nonces, 1, k2);
    const uint64_t chunk = std::min<uint64_t>(std::max<uint64_t>(count, 1), 1u << 22);
    int rc = scan.scanner(0).init(provider, challenge, nonces, pows, k1, k2, num_labels, chunk);
    if (rc) return rc;
    rc = scan.run([&](size_t, uint64_t off, uint64_t n, uint8_t *dst) {
        parallel_copy(dst, labels16 + off * 16, (size_t)n * 16);   // pageable -> pinned staging, the scan's host-side bound
        return B200POST_OK;
    }, chunk, first_index, nullptr);
    if (rc) return rc;
    uint32_t nonce = 0;
    std::vector<uint64_t> idx;
    if (!scan.rule().decide(&nonce, &idx, &rc)) return no_proof(1, nonces);
    return write_proof(scan.rule().scanned(), nonce, idx, pows, 0, num_labels, out);
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

int b200post_generate_proof_sums(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg,
                                 const b200post_prove_opts *opts, const uint32_t *providers, int n_providers,
                                 const b200post_prove_sums_opts *sopts, b200post_proof_out *out, b200post_proof_metadata *meta_out,
                                 b200post_prove_check *check, b200post_prove_sums_report *sums, const volatile int *cancel) {
    if (!data_dir || !challenge || !cfg || !out || !providers || n_providers <= 0 || !check || !sums) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    memset(check, 0, sizeof *check);
    memset(sums, 0, sizeof *sums);
    SumsCheck sc(sopts && sopts->max_heal_blocks ? sopts->max_heal_blocks : 1024);
    const int rc = generate(data_dir, challenge, cfg, opts, providers, n_providers, out, meta_out, check, cancel, &sc);
    const std::string err = rc ? last_error() : std::string();
    sums->blocks_checked = sc.blocks_checked; sums->labels_verified = sc.labels_verified; sums->labels_uncovered = sc.labels_uncovered;
    sums->bad_blocks = sc.bad.size(); sums->healed_blocks = sc.healed.size();
    for (const auto &kv : sc.bad) {   // ascending
        sums->sidecar_only += kv.second.sidecar_only;
        if (sums->n_reported < 64) sums->bad[sums->n_reported++] = b200post_sums_block{kv.first, kv.second.count};
    }
    metrics().prove_sum_blocks_checked_total += sums->blocks_checked;
    metrics().prove_sum_blocks_bad_total += sums->bad_blocks;
    metrics().prove_sum_blocks_healed_total += sums->healed_blocks;
    if (rc) set_error(err);
    return rc;
}

int b200post_generate_proofs(b200post_prove_item *items, size_t n, const b200post_post_config *cfg, const b200post_prove_opts *opts,
                             const uint32_t *providers, int n_providers, uint32_t checked, uint32_t parallel_scans,
                             const volatile int *cancel) {
    if (!items || n == 0 || !cfg || !providers || n_providers <= 0) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    for (size_t i = 0; i < n; i++)
        if (!items[i].data_dir) { set_error("invalid argument: item " + std::to_string(i) + " has no data_dir"); return B200POST_ERR_INVALID_ARGUMENT; }
    std::vector<ItemProof> its(n);
    for (size_t i = 0; i < n; i++) {
        b200post_prove_item &x = items[i];
        x.status = B200POST_OK;
        memset(x.error, 0, sizeof x.error);
        memset(&x.proof, 0, sizeof x.proof); memset(&x.meta, 0, sizeof x.meta); memset(&x.check, 0, sizeof x.check);
        its[i].data_dir = x.data_dir; its[i].challenge = x.challenge; its[i].out = &x.proof; its[i].meta_out = &x.meta;
        its[i].check = checked ? &x.check : nullptr;
    }
    const int rc = prove_items(its, *cfg, prove_opts(opts), providers, n_providers, parallel_scans, cancel);
    for (size_t i = 0; i < n; i++) {
        items[i].status = its[i].status;
        snprintf(items[i].error, sizeof items[i].error, "%s", its[i].error.c_str());
    }
    return rc;
}

}  // extern "C"

namespace {
// b200post_prove_opts with its defaults filled in
b200post_prove_opts prove_opts(const b200post_prove_opts *opts) {
    b200post_prove_opts o{};
    if (opts) o = *opts;
    if (o.nonces == 0) o.nonces = 16;
    if (o.chunk_labels == 0) o.chunk_labels = 1ull << 22;
    return o;
}

// b200post_generate_proof_multi (check == nullptr), b200post_generate_proof_checked and b200post_generate_proof_sums
// (check and sums): the one-item case of prove_items.  They differ only in the scan's hit records, whether hits are born
// pending (the ShardedScan's commitment), the chunk plan and sidecar check (sums), the report and the verifier gate.
int generate(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg, const b200post_prove_opts *opts,
             const uint32_t *providers, int n_providers, b200post_proof_out *out, b200post_proof_metadata *meta_out,
             b200post_prove_check *check, const volatile int *cancel, SumsCheck *sums) {
    std::vector<ItemProof> items(1);
    ItemProof &it = items[0];
    it.data_dir = data_dir; it.challenge = challenge; it.out = out; it.meta_out = meta_out; it.check = check; it.sums = sums;
    prove_items(items, *cfg, prove_opts(opts), providers, n_providers, 1, cancel);
    if (it.status) set_error(it.error);
    return it.status;
}
}  // namespace
