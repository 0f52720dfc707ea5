// verifier.cu — batched POST proof verification (include/b200post_verify.h).
//
// Host side of the verify path, C++ because the reference's is compiled Go
// (activation/post_verifier.go:122-390 offloadingPostVerifier + :150-160 postVerifier.Verify).  The GPU does
// what is expensive and certain — recomputing every requested label with the gather kernels — and this file
// does the cheap per-proof bookkeeping around it.  All conventions marked ASSUMED follow the published
// post-rs v0.7.x verifier from memory and are "parity unpinned" (DESIGN.md §2).
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <map>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/b200post_verify.h"
#include "aes_device.cuh"
#include "engine.h"
#include "host_hash.h"
#include "metrics.h"
#include "proof_common.h"
#include "randomx_engine.h"
#include "../../include/b200post_k2pow.h"

namespace b200post {
namespace {

// ASSUMED (post-rs random_values_gen.rs): BLAKE3-XOF driven partial Fisher-Yates over the K2 positions.
struct Blake3Rng {
    std::vector<uint8_t> seed;
    std::vector<uint8_t> buf;
    size_t pos = 0;
    bool ok = true;
    explicit Blake3Rng(std::vector<uint8_t> s) : seed(std::move(s)) { refill(256); }
    void refill(size_t n) {
        buf.resize(n);
        ok = blake3_single_chunk(seed.data(), seed.size(), buf.data(), n);
    }
    uint16_t next_u16() {
        if (pos + 2 > buf.size()) refill(buf.size() * 2);   // XOF output is a prefix-stable stream
        const uint16_t v = (uint16_t)(buf[pos] | (buf[pos + 1] << 8));
        pos += 2;
        return v;
    }
};

// One queue entry: a proof, or (vrf != nullptr) a VRF-nonce check.  Both kinds share the queues and the batch; a
// VRF check is one label (the one at its nonce), judged by K9 instead of K5, and never reaches the k2pow step.
struct Job {
    const b200post_proof *proof = nullptr;
    const b200post_proof_metadata *meta = nullptr;
    const b200post_verify_params *params = nullptr;
    const b200post_vrf_check *vrf = nullptr;
    b200post_verify_options opt;
    int status = B200POST_OK;
    uint64_t bad_index = 0;
    bool done = false;
    // filled by prepare()
    std::vector<uint64_t> check;   // label indices to recompute, in verification order
    std::vector<uint32_t> pos;     // position of each of them in the proof's K2 index list (what ErrInvalidIndex reports)
    uint64_t bad_label = 0;        // the label index stored at the failing position
    uint8_t pow_input[48];         // k2pow input of this proof (builtin pow check)
    uint8_t pow_target[32];        // pow_difficulty / num_units
    uint8_t commitment[32];
    uint8_t key[16], lazy_key[16];
    uint8_t diff_msb = 0;
    uint64_t diff_lsb = 0;
    uint32_t out_byte = 0;
    size_t first_item = 0;
    // VRF check: threshold floor(2^256 / numLabels) as big-endian words (filled by prepare()), and the results
    uint32_t vrf_threshold[8];
    int vrf_valid = 0;
    uint8_t label32[32] = {0};
    uint64_t scrypt_n() const { return vrf ? vrf->scrypt_n : params->scrypt_n; }
};

}  // namespace
}  // namespace b200post

using namespace b200post;

extern "C" {

uint32_t b200post_bits_per_index(uint64_t num_labels) {
    // ASSUMED: floor(log2(n)) + 1  (post-rs compression::required_bits / Go shared.BinaryRepresentationMinBits)
    return num_labels == 0 ? 0 : 64 - (uint32_t)__builtin_clzll(num_labels);
}

uint64_t b200post_proving_difficulty(uint32_t k1, uint64_t num_labels) {
    // ASSUMED: floor(2^64 * k1 / num_labels), saturating
    if (num_labels == 0) return 0;
    const unsigned __int128 v = ((unsigned __int128)k1 << 64) / num_labels;
    return v > (unsigned __int128)~0ull ? ~0ull : (uint64_t)v;
}

size_t b200post_pack_indices(const uint64_t *indices, size_t count, uint32_t bits, uint8_t *out, size_t out_cap) {
    const size_t need = (count * (size_t)bits + 7) / 8;
    if (!out || out_cap < need || bits == 0 || bits > 64) return 0;
    memset(out, 0, need);
    size_t bitpos = 0;
    for (size_t i = 0; i < count; i++)
        for (uint32_t j = 0; j < bits; j++, bitpos++)
            if ((indices[i] >> j) & 1) out[bitpos >> 3] |= (uint8_t)(1u << (bitpos & 7));
    return need;
}

size_t b200post_unpack_indices(const uint8_t *packed, size_t packed_len, uint32_t bits, uint64_t *out, size_t out_cap) {
    if (!packed || !out || bits == 0 || bits > 64) return 0;
    const size_t n = std::min(out_cap, packed_len * 8 / bits);
    size_t bitpos = 0;
    for (size_t i = 0; i < n; i++) {
        uint64_t v = 0;
        for (uint32_t j = 0; j < bits; j++, bitpos++) v |= (uint64_t)((packed[bitpos >> 3] >> (bitpos & 7)) & 1) << j;
        out[i] = v;
    }
    return n;
}

int b200post_verify_batch_multi(const uint32_t *providers, int n_providers, size_t n, const b200post_proof *proofs,
                                const b200post_proof_metadata *metas, const b200post_verify_params *params,
                                const b200post_verify_options *options, const b200post_verifier_opts *opts, int *statuses,
                                uint64_t *invalid_indices) {
    if (!providers || n_providers <= 0) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    if (n_providers == 1 || n < 2) return b200post_verify_batch(providers[0], n, proofs, metas, params, options, opts, statuses, invalid_indices);
    if (int rc = device_engines(providers, n_providers)) return rc;
    const size_t parts = std::min<size_t>((size_t)n_providers, n);
    return fan_out(parts, [=](size_t d) {
        const size_t lo = n * d / parts, hi = n * (d + 1) / parts;
        return b200post_verify_batch(providers[d], hi - lo, proofs + lo, metas + lo, params, options ? options + lo : nullptr, opts,
                                     statuses + lo, invalid_indices ? invalid_indices + lo : nullptr);
    });
}

}  // extern "C"

namespace b200post {
namespace {

// A VRF check's host part: its numLabels, threshold and commitment; the one label to recompute is at the nonce.  The
// nonce is not range-checked: a nonce >= numLabels is what the past-the-end search produces.
void prepare_vrf(Job &j) {
    const b200post_vrf_check &c = *j.vrf;
    j.status = B200POST_OK;
    const unsigned __int128 nl = (unsigned __int128)c.num_units * c.labels_per_unit;
    if (nl == 0 || nl > ~0ull) { j.status = B200POST_ERR_INVALID_ARGUMENT; return; }
    uint8_t diff[32];
    vrf_difficulty((uint64_t)nl, diff);
    for (int k = 0; k < 8; k++)
        j.vrf_threshold[k] = ((uint32_t)diff[4 * k] << 24) | ((uint32_t)diff[4 * k + 1] << 16) | ((uint32_t)diff[4 * k + 2] << 8) | diff[4 * k + 3];
    commitment_bytes(c.node_id, c.commitment_atx_id, j.commitment);
    j.check.assign(1, c.nonce);
}

// Per-proof checks that need no labels; fills job.check with the label indices to recompute.
void prepare(Job &j, const b200post_verifier_opts &vo) {
    if (j.vrf) { prepare_vrf(j); return; }
    const b200post_proof &p = *j.proof;
    const b200post_proof_metadata &m = *j.meta;
    const b200post_verify_params &q = *j.params;
    j.status = B200POST_OK;
    if (!p.indices || p.indices_len == 0) { j.status = B200POST_ERR_EMPTY_PROOF; return; }   // "proof indices are empty"
    const unsigned __int128 nl = (unsigned __int128)m.num_units * m.labels_per_unit;
    // k2 <= 65535: the Subset shuffle draws 16-bit values (and the wire format caps a proof at 800 bytes anyway,
    // activation/wire/wire_v1.go:41-45)
    if (nl == 0 || nl > ~0ull || q.k2 == 0 || q.k2 > 0xffffu || q.k1 == 0 || m.num_units == 0) { j.status = B200POST_ERR_INVALID_ARGUMENT; return; }
    const uint64_t num_labels = (uint64_t)nl;
    const uint32_t bits = b200post_bits_per_index(num_labels);
    const size_t expect_len = ((size_t)q.k2 * bits + 7) / 8;
    if (p.indices_len != expect_len) { j.status = B200POST_ERR_INVALID_ARGUMENT; return; }   // wrong number of indices
    const uint32_t nonce_group = p.nonce / 16;
    if (vo.pow_mode != B200POST_POW_SKIP) {
        if (nonce_group > 255) { j.status = B200POST_ERR_INVALID_ARGUMENT; return; }
        div256_u32(q.pow_difficulty, m.num_units, j.pow_target);
        if (vo.pow_mode == B200POST_POW_CALLBACK) {
            if (vo.pow_verify(vo.pow_ctx, p.pow, (uint8_t)nonce_group, m.challenge, j.pow_target, m.node_id) != 0) {
                j.status = B200POST_ERR_INVALID_PROOF;
                j.bad_index = ~0ull;   // the pow, not a label, is invalid
                return;
            }
        } else {
            // builtin: the RandomX hashes of the whole batch are computed together on the device (process())
            if (p.pow >> 56) { j.status = B200POST_ERR_INVALID_PROOF; j.bad_index = ~0ull; return; }   // more than the 7 bytes the prover hashes
            for (int b = 0; b < 7; b++) j.pow_input[b] = (uint8_t)(p.pow >> (8 * b));
            j.pow_input[7] = (uint8_t)nonce_group;
            memcpy(j.pow_input + 8, m.challenge, 8);
            memcpy(j.pow_input + 16, m.node_id, 32);
        }
    }
    std::vector<uint64_t> all(q.k2);
    std::vector<uint32_t> where(q.k2);
    for (uint32_t i = 0; i < q.k2; i++) where[i] = i;
    if (b200post_unpack_indices(p.indices, p.indices_len, bits, all.data(), all.size()) != q.k2) { j.status = B200POST_ERR_INVALID_ARGUMENT; return; }
    switch (j.opt.mode) {
        case B200POST_VERIFY_ALL: j.check = std::move(all); j.pos = std::move(where); break;
        case B200POST_VERIFY_SELECTED_INDEX:
            if (j.opt.selected_index >= q.k2) { j.status = B200POST_ERR_INVALID_ARGUMENT; return; }
            j.check.assign(1, all[j.opt.selected_index]);
            j.pos.assign(1, j.opt.selected_index);
            break;
        case B200POST_VERIFY_SUBSET: {
            const uint32_t k3 = std::min(j.opt.k3, q.k2);
            if (k3 == 0) { j.status = B200POST_ERR_INVALID_ARGUMENT; return; }
            // seed = caller seed || LE32(nonce) || indices || LE64(pow)   — ASSUMED
            std::vector<uint8_t> seed;
            if (j.opt.seed && j.opt.seed_len) seed.assign(j.opt.seed, j.opt.seed + j.opt.seed_len);
            uint8_t tmp[8];
            put_le32(tmp, p.nonce); seed.insert(seed.end(), tmp, tmp + 4);
            seed.insert(seed.end(), p.indices, p.indices + p.indices_len);
            put_le64(tmp, p.pow); seed.insert(seed.end(), tmp, tmp + 8);
            if (seed.size() > 1024) { j.status = B200POST_ERR_INVALID_ARGUMENT; return; }
            Blake3Rng rng(std::move(seed));
            size_t idx = 0;
            while (j.check.size() < k3 && idx < all.size()) {
                const uint16_t remaining = (uint16_t)(all.size() - idx);
                const uint16_t max_allowed = (uint16_t)(0xffffu - 0xffffu % remaining);
                uint16_t r;
                do { r = rng.next_u16(); } while (r >= max_allowed && rng.ok);
                if (!rng.ok) { j.status = B200POST_ERR_INVALID_ARGUMENT; return; }
                std::swap(all[idx], all[idx + r % remaining]);
                std::swap(where[idx], where[idx + r % remaining]);
                j.check.push_back(all[idx]);
                j.pos.push_back(where[idx]);
                idx++;
            }
            break;
        }
        default: j.status = B200POST_ERR_INVALID_ARGUMENT; return;
    }
    // indices >= num_labels are not rejected here: as upstream, the label is simply recomputed and judged
    commitment_bytes(m.node_id, m.commitment_atx_id, j.commitment);
    cipher_key(m.challenge, nonce_group, p.pow, nullptr, j.key);
    cipher_key(m.challenge, nonce_group, p.pow, &p.nonce, j.lazy_key);
    const uint64_t diff = b200post_proving_difficulty(q.k1, num_labels);
    j.diff_msb = (uint8_t)(diff >> 56);
    j.diff_lsb = diff & 0x00ffffffffffffffull;
    j.out_byte = p.nonce % 16;
}

// ---------------------------------------------------------------------------------------------- device epilogue
// K5 verify_judge_kernel: the label-dependent verdict, on the device, straight from the labels K3 left in
// HBM (no label D2H, no host AES).  One thread per recomputed label: AES-128 under the proof's key, compare
// ciphertext byte (nonce mod 16) with the top 8 bits of the proving difficulty; on equality the lazy cipher
// decides with the low 56 bits.  The first failing position per proof is kept with atomicMin.
struct DevJob {            // 384 bytes
    uint4 rk[11];
    uint4 lazy_rk[11];
    uint32_t first_item, n_items, out_byte, diff_msb;
    uint64_t diff_lsb;
    uint32_t pad[2];
};

__global__ void __launch_bounds__(256) verify_judge_kernel(const uint4 *__restrict__ labels, const uint32_t *__restrict__ item_job,
                                                           const DevJob *__restrict__ jobs, uint32_t n_items,
                                                           const AesTables *__restrict__ tables, uint32_t *__restrict__ first_bad) {
    extern __shared__ uint32_t aes_sm[];
    aes_load_smem(aes_sm, tables);
    const uint32_t *tl = aes_sm + (threadIdx.x & 31);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_items) return;
    const uint32_t jb = item_job[i];
    const DevJob &j = jobs[jb];
    const uint4 label = labels[i];
    uint4 out = aes128_encrypt(tl, j.rk, label);
    const uint32_t msb = uint4_byte(out, j.out_byte);
    bool bad = msb > j.diff_msb;
    if (msb == j.diff_msb) {
        out = aes128_encrypt(tl, j.lazy_rk, label);
        const uint64_t lsb = ((uint64_t)out.x | ((uint64_t)out.y << 32)) & 0x00ffffffffffffffull;
        bad = lsb >= j.diff_lsb;
    }
    if (bad) atomicMin(&first_bad[jb], i - j.first_item);
}

// run fn(i) for i in [0, n) on up to 16 host threads (the per-proof prologue/epilogue is independent work)
template <typename F>
void parallel_for(size_t n, F fn) {
    const size_t nt = std::min<size_t>({(size_t)16, std::max<size_t>(1, std::thread::hardware_concurrency()), (n + 255) / 256});
    if (nt <= 1) { for (size_t i = 0; i < n; i++) fn(i); return; }
    std::vector<std::thread> th;
    for (size_t t = 0; t < nt; t++)
        th.emplace_back([=] { for (size_t i = t; i < n; i += nt) fn(i); });
    for (auto &x : th) x.join();
}

// Recompute the labels of all OK jobs with scrypt-N `n` (gather kernels, labels stay in HBM) and run the
// device epilogue.  first_bad[k] = position of the first failing label of the k-th such job, or 0xffffffff.
// grow-only device buffers of the judge stage, one set per provider: a batch costs no cudaMalloc/cudaFree once warm
struct JudgeScratch {
    std::mutex mu;
    DeviceBuffer<uint4> labels;
    DeviceBuffer<uint32_t> item_job, first_bad;
    DeviceBuffer<DevJob> jobs;
    DeviceBuffer<AesTables> tables;
    // VRF checks: the high label halves of the gather (K3w), and per check the threshold, K9's verdict and label32
    DeviceBuffer<uint4> labels_hi, vrf_threshold, vrf_label;
    DeviceBuffer<uint8_t> vrf_valid;
    int reserve_vrf(size_t n_items, size_t n_vrf) {
        if (n_items > labels_hi.size()) CUDA_TRY(labels_hi.resize(n_items + n_items / 4));
        if (n_vrf > vrf_valid.size()) {   // vrf_valid is allocated last: its size is the capacity of all three
            vrf_valid.reset();
            const size_t c = n_vrf + n_vrf / 4;
            CUDA_TRY(vrf_threshold.resize(2 * c));
            CUDA_TRY(vrf_label.resize(2 * c));
            CUDA_TRY(vrf_valid.resize(c));
        }
        return B200POST_OK;
    }
    int reserve(size_t n_items, size_t n_jobs, const AesTables &host_tables) {
        if (!tables.get()) {
            CUDA_TRY(tables.resize(1));
            CUDA_TRY(cudaMemcpy(tables.get(), &host_tables, sizeof(AesTables), cudaMemcpyHostToDevice));
        }
        if (n_items > item_job.size()) {   // item_job is allocated last: its size is the capacity of both
            item_job.reset();
            const size_t c = n_items + n_items / 4;
            CUDA_TRY(labels.resize(c));
            CUDA_TRY(item_job.resize(c));
        }
        if (n_jobs > first_bad.size()) {   // likewise first_bad
            first_bad.reset();
            const size_t c = n_jobs + n_jobs / 4;
            CUDA_TRY(jobs.resize(c));
            CUDA_TRY(first_bad.resize(c));
        }
        return B200POST_OK;
    }
};
JudgeScratch &judge_scratch(uint32_t provider) {
    static std::mutex mu;
    static std::map<uint32_t, JudgeScratch *> *all = new std::map<uint32_t, JudgeScratch *>;   // never destroyed: the CUDA context may be gone at exit
    std::lock_guard<std::mutex> lk(mu);
    JudgeScratch *&s = (*all)[provider];
    if (!s) s = new JudgeScratch;
    return *s;
}

// `indices` holds every checked label index of the batch, proof after proof, then one per VRF check (Job::first_item);
// each job's commitment is uploaded once and items refer to it by row (DeviceEngine::labels_gather_indexed): the
// proofs' rows first, so that a proof item's row is also its DevJob.  K5 judges the proof items; when VRF checks are
// present the gather keeps both label halves (K3w) and K9 judges the checks, whose results land in their jobs.
int gather_and_judge(uint32_t provider, const std::vector<Job *> &live, const std::vector<Job *> &vrfs, uint64_t n,
                     const std::vector<uint64_t> &indices, std::vector<uint32_t> &first_bad) {
    DeviceEngine *e = engine_for(provider);
    if (!e) return B200POST_ERR_NO_DEVICE;
    std::vector<DevJob> dj(live.size());
    std::vector<uint8_t> commitments((live.size() + vrfs.size()) * 32);
    std::vector<uint32_t> item_job(indices.size());
    std::vector<uint32_t> thresholds(vrfs.size() * 8);
    for (size_t v = 0; v < vrfs.size(); v++) {
        const size_t row = live.size() + v;
        memcpy(&commitments[row * 32], vrfs[v]->commitment, 32);
        item_job[vrfs[v]->first_item] = (uint32_t)row;
        memcpy(&thresholds[v * 8], vrfs[v]->vrf_threshold, 32);
    }
    parallel_for(live.size(), [&](size_t i) {
        Job *j = live[i];
        DevJob &d = dj[i];
        memset(&d, 0, sizeof d);
        const Aes128 a(j->key), l(j->lazy_key);
        memcpy(d.rk, a.rk, sizeof d.rk);
        memcpy(d.lazy_rk, l.rk, sizeof d.lazy_rk);
        d.first_item = (uint32_t)j->first_item; d.n_items = (uint32_t)j->check.size();
        d.out_byte = j->out_byte; d.diff_msb = j->diff_msb; d.diff_lsb = j->diff_lsb;
        memcpy(&commitments[i * 32], j->commitment, 32);
        for (size_t k = 0; k < j->check.size(); k++) item_job[j->first_item + k] = (uint32_t)i;
    });
    first_bad.assign(dj.size(), 0xffffffffu);
    if (indices.empty()) return B200POST_OK;
    static AesTables host_tables;
    static std::once_flag once;
    std::call_once(once, [] { aes_build_tables(host_tables); });

    const uint32_t n_items = (uint32_t)indices.size();
    const uint32_t n_vrf = (uint32_t)vrfs.size(), n_proof_items = n_items - n_vrf;
    CUDA_TRY(cudaSetDevice(e->device()));
    JudgeScratch &s = judge_scratch(provider);
    std::lock_guard<std::mutex> lk(s.mu);
    int rc = s.reserve(n_items, dj.size(), host_tables);
    if (rc == B200POST_OK && n_vrf) rc = s.reserve_vrf(n_items, n_vrf);
    if (rc != B200POST_OK) return rc;
    CUDA_TRY(cudaMemcpy(s.item_job.get(), item_job.data(), (size_t)n_items * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(s.jobs.get(), dj.data(), dj.size() * sizeof(DevJob), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemset(s.first_bad.get(), 0xff, dj.size() * 4));
    if (n_vrf) CUDA_TRY(cudaMemcpy(s.vrf_threshold.get(), thresholds.data(), thresholds.size() * 4, cudaMemcpyHostToDevice));
    rc = e->labels_gather_indexed(indices.size(), live.size() + n_vrf, commitments.data(), item_job.data(), indices.data(), n, nullptr,
                                  reinterpret_cast<uint8_t *>(s.labels.get()),
                                  n_vrf ? reinterpret_cast<uint8_t *>(s.labels_hi.get()) : nullptr);
    if (rc != B200POST_OK) return rc;
    if (n_proof_items) {
        verify_judge_kernel<<<(n_proof_items + 255) / 256, 256, AES_SMEM_BYTES>>>(s.labels.get(), s.item_job.get(), s.jobs.get(),
                                                                                  n_proof_items, s.tables.get(), s.first_bad.get());
        g_launches += 1;
        CUDA_TRY(cudaGetLastError());
    }
    if (n_vrf) {
        CUDA_TRY(launch_vrf_judge(s.labels.get(), s.labels_hi.get(), n_proof_items, n_vrf, s.vrf_threshold.get(), s.vrf_valid.get(),
                                  s.vrf_label.get(), 0));
        g_launches += 1;
        std::vector<uint8_t> valid(n_vrf), label32((size_t)n_vrf * 32);
        CUDA_TRY(cudaMemcpy(valid.data(), s.vrf_valid.get(), n_vrf, cudaMemcpyDeviceToHost));
        CUDA_TRY(cudaMemcpy(label32.data(), s.vrf_label.get(), label32.size(), cudaMemcpyDeviceToHost));
        for (uint32_t v = 0; v < n_vrf; v++) {
            vrfs[v]->vrf_valid = valid[v];
            memcpy(vrfs[v]->label32, &label32[(size_t)v * 32], 32);
        }
    }
    CUDA_TRY(cudaMemcpy(first_bad.data(), s.first_bad.get(), dj.size() * 4, cudaMemcpyDeviceToHost));
    return B200POST_OK;
}

// One GPU batch: jobs may use different scrypt N; group by N (in practice a single value).
int process(uint32_t provider, std::vector<Job *> &jobs, const b200post_verifier_opts &vo) {
    const auto t0 = std::chrono::steady_clock::now();
    if (vo.pow_mode == B200POST_POW_CALLBACK) { for (Job *j : jobs) prepare(*j, vo); }   // the callback's thread-safety is the caller's business
    else parallel_for(jobs.size(), [&](size_t i) { prepare(*jobs[i], vo); });
    if (vo.pow_mode == B200POST_POW_BUILTIN) {
        // the k2pow check of verifying.ProofVerifier.Verify (activation/post_verifier.go:150-160): one RandomX hash per
        // proof, all proofs of the batch in one device batch.  VRF checks have no pow: a batch of only VRF checks never
        // touches the RandomX engine (nor builds its dataset).
        std::vector<Job *> live;
        for (Job *j : jobs) if (j->status == B200POST_OK && !j->vrf) live.push_back(j);
        if (!live.empty()) {
            std::vector<uint8_t> in(live.size() * 48), out(live.size() * 32);
            for (size_t i = 0; i < live.size(); i++) memcpy(&in[i * 48], live[i]->pow_input, 48);
            RandomxEngine *rxe = randomx_engine_for(provider);
            const std::string key = vo.pow_cache_key ? std::string(reinterpret_cast<const char *>(vo.pow_cache_key), vo.pow_cache_key_len)
                                                     : std::string(B200POST_K2POW_DEFAULT_KEY);
            const int rc = rxe ? rxe->hash_inputs(key, in.data(), 48, live.size(), out.data()) : B200POST_ERR_NO_DEVICE;
            for (size_t i = 0; i < live.size(); i++) {
                if (rc != B200POST_OK) live[i]->status = rc;
                else if (memcmp(&out[i * 32], live[i]->pow_target, 32) >= 0) { live[i]->status = B200POST_ERR_INVALID_PROOF; live[i]->bad_index = ~0ull; }
            }
        }
    }
    const auto t1 = std::chrono::steady_clock::now();
    metrics().verify_prepare_us_total += (uint64_t)std::chrono::duration_cast<std::chrono::microseconds>(t1 - t0).count();
    struct Stage { std::chrono::steady_clock::time_point from; ~Stage() {
        metrics().verify_gather_judge_us_total += (uint64_t)std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - from).count(); } } stage{t1};
    std::vector<uint64_t> ns;
    for (Job *j : jobs)
        if (j->status == B200POST_OK && std::find(ns.begin(), ns.end(), j->scrypt_n()) == ns.end()) ns.push_back(j->scrypt_n());
    for (uint64_t n : ns) {
        // one gather per N: the proofs' labels, then one label per VRF check
        std::vector<Job *> live, vrfs;
        size_t total = 0;
        for (Job *j : jobs) {
            if (j->status != B200POST_OK || j->scrypt_n() != n) continue;
            (j->vrf ? vrfs : live).push_back(j);
            total += j->check.size();
        }
        std::vector<uint64_t> indices;
        indices.reserve(total);
        for (Job *j : live) {
            j->first_item = indices.size();
            indices.insert(indices.end(), j->check.begin(), j->check.end());
        }
        for (Job *j : vrfs) {
            j->first_item = indices.size();
            indices.push_back(j->check[0]);
        }
        int rc = B200POST_ERR_INVALID_ARGUMENT;
        std::vector<uint32_t> first_bad;
        if (n >= 2 && n <= (1ull << 20) && (n & (n - 1)) == 0) rc = gather_and_judge(provider, live, vrfs, n, indices, first_bad);
        for (Job *j : vrfs) if (rc != B200POST_OK) j->status = rc;
        size_t k = 0;
        for (Job *j : live) {
            if (rc != B200POST_OK) j->status = rc;
            else if (first_bad[k] != 0xffffffffu) {
                // verifying.ErrInvalidIndex{Index}: the POSITION in the proof's K2 list (activation/handler_v1.go:248 stores it as
                // InvalidPostIndexProof.InvalidIdx, activation/malfeasance.go:165 re-verifies it with SelectedIndex(InvalidIdx))
                j->status = B200POST_ERR_INVALID_PROOF; j->bad_index = j->pos[first_bad[k]]; j->bad_label = j->check[first_bad[k]];
            }
            k++;
        }
    }
    return B200POST_OK;
}

}  // namespace
}  // namespace b200post

struct b200post_verifier {
    uint32_t provider = 0;
    b200post_verifier_opts opts{};
    std::mutex mu;
    std::condition_variable cv_work, cv_done;
    std::deque<Job *> prioritized, normal;
    bool closed = false;
    uint64_t batches = 0, proofs = 0;
    std::vector<std::thread> workers;     // one per device; all drain the same two queues

    void run(uint32_t provider) {
        std::unique_lock<std::mutex> lk(mu);
        for (;;) {
            cv_work.wait(lk, [&] { return closed || !prioritized.empty() || !normal.empty(); });
            if (closed) {
                for (auto *q : {&prioritized, &normal}) {
                    for (Job *j : *q) { j->status = B200POST_ERR_CLOSED; j->done = true; }
                    q->clear();
                }
                cv_done.notify_all();
                return;
            }
            // drain everything queued (prioritised first): while the GPU works on this batch the next one fills
            std::vector<Job *> batch;
            // several devices: leave the others their share of a long queue, but do not shred a short one
            size_t cap = opts.max_batch_proofs ? opts.max_batch_proofs : 16384;
            if (workers.size() > 1) {
                const size_t queued = prioritized.size() + normal.size();
                cap = std::min(cap, std::max<size_t>(64, (queued + workers.size() - 1) / workers.size()));
            }
            while (batch.size() < cap && !prioritized.empty()) { batch.push_back(prioritized.front()); prioritized.pop_front(); }
            while (batch.size() < cap && !normal.empty()) { batch.push_back(normal.front()); normal.pop_front(); }
            lk.unlock();
            process(provider, batch, opts);
            lk.lock();
            batches++;
            for (Job *j : batch) proofs += j->vrf ? 0 : 1;   // VRF checks are not proofs
            metrics().verify_batches_total++;
            for (Job *j : batch) j->done = true;
            cv_done.notify_all();
        }
    }
};

extern "C" {

int b200post_verifier_new(uint32_t provider, const b200post_verifier_opts *opts, b200post_verifier **out) {
    if (!out) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    *out = nullptr;
    if (int rc = device_engine(provider)) return rc;
    return b200post_verifier_new_multi(&provider, 1, opts, out);
}

int b200post_verifier_new_multi(const uint32_t *providers, int n_providers, const b200post_verifier_opts *opts,
                                b200post_verifier **out) {
    if (!out || !providers || n_providers <= 0) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    *out = nullptr;
    if (int rc = device_engines(providers, n_providers)) return rc;
    if (opts && (opts->pow_mode > B200POST_POW_SKIP || (opts->pow_mode == B200POST_POW_CALLBACK && !opts->pow_verify))) {
        set_error("pow_mode CALLBACK needs a pow_verify function; to run without the k2pow check ask for B200POST_POW_SKIP explicitly");
        return B200POST_ERR_UNSUPPORTED;
    }
    b200post_verifier *v = new b200post_verifier;
    v->provider = providers[0];
    if (opts) v->opts = *opts;
    v->workers.reserve((size_t)n_providers);     // run() reads workers.size(): no reallocation while threads start
    {
        std::lock_guard<std::mutex> lk(v->mu);
        for (int d = 0; d < n_providers; d++) { const uint32_t p = providers[d]; v->workers.emplace_back([v, p] { v->run(p); }); }
    }
    *out = v;
    return B200POST_OK;
}

int b200post_verifier_verify(b200post_verifier *v, const b200post_proof *proof, const b200post_proof_metadata *meta,
                             const b200post_verify_params *params, const b200post_verify_options *options,
                             uint64_t *invalid_index) {
    if (!v || !proof || !meta || !params) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    Job j;
    j.proof = proof; j.meta = meta; j.params = params;
    if (options) j.opt = *options; else memset(&j.opt, 0, sizeof j.opt);
    const auto t_begin = std::chrono::steady_clock::now();
    metrics().verify_waiting++;                       // metrics.PostVerificationQueue.Inc() (post_verifier.go:319)
    struct Leave { ~Leave() { metrics().verify_waiting--; } } leave;
    {
        std::unique_lock<std::mutex> lk(v->mu);
        if (v->closed) { set_error("verifier is closed"); return B200POST_ERR_CLOSED; }
        (j.opt.prioritized ? v->prioritized : v->normal).push_back(&j);
        v->cv_work.notify_one();
        v->cv_done.wait(lk, [&] { return j.done; });
    }
    if (j.status == B200POST_ERR_CLOSED) set_error("verifier is closed");
    else if (j.status == B200POST_ERR_EMPTY_PROOF) set_error("proof indices are empty");
    else if (j.status == B200POST_ERR_INVALID_PROOF) set_error(j.bad_index == ~0ull ? "invalid k2pow" : "invalid index");
    else if (j.status == B200POST_ERR_INVALID_ARGUMENT) set_error("malformed proof, metadata or options");
    if (invalid_index) *invalid_index = j.bad_index;
    if (j.status != B200POST_ERR_CLOSED) {
        metrics().verify_proofs_total++;
        if (j.status == B200POST_ERR_INVALID_PROOF) metrics().verify_invalid_total++;
        observe_verify_seconds(std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count());
    }
    return j.status;
}

int b200post_verifier_verify_vrf_nonce(b200post_verifier *v, const b200post_vrf_check *c, int *valid, uint8_t label32[32]) {
    if (!v || !c || !valid) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    *valid = 0;
    Job j;
    j.vrf = c;
    memset(&j.opt, 0, sizeof j.opt);
    {
        std::unique_lock<std::mutex> lk(v->mu);
        if (v->closed) { set_error("verifier is closed"); return B200POST_ERR_CLOSED; }
        (c->prioritized ? v->prioritized : v->normal).push_back(&j);
        v->cv_work.notify_one();
        v->cv_done.wait(lk, [&] { return j.done; });
    }
    if (j.status == B200POST_ERR_CLOSED) set_error("verifier is closed");
    else if (j.status == B200POST_ERR_INVALID_ARGUMENT) set_error("malformed VRF check (num_units * labels_per_unit or scrypt N)");
    if (j.status != B200POST_OK) return j.status;
    *valid = j.vrf_valid;
    if (label32) memcpy(label32, j.label32, 32);
    return B200POST_OK;
}

int b200post_verifier_close(b200post_verifier *v) {
    if (!v) return B200POST_ERR_INVALID_ARGUMENT;
    {
        std::lock_guard<std::mutex> lk(v->mu);
        if (v->closed) return B200POST_OK;
        v->closed = true;
    }
    v->cv_work.notify_all();
    for (auto &w : v->workers) if (w.joinable()) w.join();
    return B200POST_OK;
}

void b200post_verifier_free(b200post_verifier *v) {
    if (!v) return;
    b200post_verifier_close(v);
    delete v;
}

int b200post_verifier_stats(b200post_verifier *v, uint64_t *batches, uint64_t *proofs) {
    if (!v) return B200POST_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> lk(v->mu);
    if (batches) *batches = v->batches;
    if (proofs) *proofs = v->proofs;
    return B200POST_OK;
}

int b200post_verify_batch(uint32_t provider, size_t n, const b200post_proof *proofs, const b200post_proof_metadata *metas,
                          const b200post_verify_params *params, const b200post_verify_options *options,
                          const b200post_verifier_opts *opts, int *statuses, uint64_t *invalid_indices) {
    if (n && (!proofs || !metas || !params || !statuses)) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    if (int rc = device_engine(provider)) return rc;
    b200post_verifier_opts vo{};
    if (opts) vo = *opts;
    if (vo.pow_mode > B200POST_POW_SKIP || (vo.pow_mode == B200POST_POW_CALLBACK && !vo.pow_verify)) {
        set_error("pow_mode CALLBACK needs a pow_verify function; to run without the k2pow check ask for B200POST_POW_SKIP explicitly");
        return B200POST_ERR_UNSUPPORTED;
    }
    std::vector<Job> jobs(n);
    std::vector<Job *> ptrs(n);
    for (size_t i = 0; i < n; i++) {
        jobs[i].proof = &proofs[i]; jobs[i].meta = &metas[i]; jobs[i].params = params;
        if (options) jobs[i].opt = options[i]; else memset(&jobs[i].opt, 0, sizeof jobs[i].opt);
        ptrs[i] = &jobs[i];
    }
    process(provider, ptrs, vo);
    metrics().verify_batches_total++; metrics().verify_proofs_total += n;
    for (size_t i = 0; i < n; i++) {
        if (jobs[i].status == B200POST_ERR_INVALID_PROOF) metrics().verify_invalid_total++;
        statuses[i] = jobs[i].status;
        if (invalid_indices) invalid_indices[i] = jobs[i].bad_index;
    }
    return B200POST_OK;
}

int b200post_verify_vrf_nonces(uint32_t provider, size_t n, const b200post_vrf_check *checks, int *statuses, int *valid,
                               uint8_t *labels32) {
    if (n && (!checks || !statuses || !valid)) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    if (int rc = device_engine(provider)) return rc;
    if (n == 0) return B200POST_OK;
    std::vector<Job> jobs(n);
    std::vector<Job *> ptrs(n);
    for (size_t i = 0; i < n; i++) {
        jobs[i].vrf = &checks[i];
        memset(&jobs[i].opt, 0, sizeof jobs[i].opt);
        ptrs[i] = &jobs[i];
    }
    b200post_verifier_opts vo{};
    vo.pow_mode = B200POST_POW_SKIP;   // VRF checks have no pow; nothing reads it
    process(provider, ptrs, vo);
    metrics().verify_batches_total++;
    for (size_t i = 0; i < n; i++) {
        statuses[i] = jobs[i].status;
        valid[i] = jobs[i].status == B200POST_OK ? jobs[i].vrf_valid : 0;
        if (labels32) {
            if (jobs[i].status == B200POST_OK) memcpy(labels32 + 32 * i, jobs[i].label32, 32);
            else memset(labels32 + 32 * i, 0, 32);
        }
    }
    return B200POST_OK;
}

int b200post_verify_vrf_nonces_multi(const uint32_t *providers, int n_providers, size_t n, const b200post_vrf_check *checks,
                                     int *statuses, int *valid, uint8_t *labels32) {
    if (!providers || n_providers <= 0 || (n && (!checks || !statuses || !valid))) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    if (int rc = device_engines(providers, n_providers)) return rc;
    if (n_providers == 1 || n < 2) return b200post_verify_vrf_nonces(providers[0], n, checks, statuses, valid, labels32);
    const size_t parts = std::min<size_t>((size_t)n_providers, n);
    return fan_out(parts, [=](size_t d) {
        const size_t lo = n * d / parts, hi = n * (d + 1) / parts;
        return b200post_verify_vrf_nonces(providers[d], hi - lo, checks + lo, statuses + lo, valid + lo,
                                          labels32 ? labels32 + 32 * lo : nullptr);
    });
}

}  // extern "C"
