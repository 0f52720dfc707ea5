// prove_internal.h — the prover's pieces that the setup session's initial proof (setup.cu, initial_proof.cu) reuses:
// the streaming scan (Scanner: K6a/K6b behind double-buffered pinned staging), the selection rule, the proof record,
// the k2pow step and the verifier gate.  Defined in prover.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <map>
#include <mutex>
#include <vector>

#include "../../include/b200post_prove.h"
#include "aes_device.cuh"
#include "engine.h"

namespace b200post {

// nonce -> its first hit indices (at most K2), ascending; ordered, so ties resolve to the lower nonce
using HitLists = std::map<uint32_t, std::vector<uint64_t>>;

// The selection rule, for one scan and for the merge of several: among nonces with K2 hits, the lowest K2-th hit
// index wins; ties go to the lower nonce.
bool pick_winner(const HitLists &lists, uint32_t k2, uint32_t *nonce, std::vector<uint64_t> *indices);

// A hit the checked scan keeps: its stored bytes, and whether they have been recomputed and found equal (good) or
// not yet looked at (pending).  A damaged hit is removed from its list.
struct KeptHit { uint64_t index; uint8_t label[16]; bool good; };
using KeptLists = std::map<uint32_t, std::vector<KeptHit>>;   // nonce -> every kept hit, ascending index

// Streaming scan state: device buffers, keys, per-nonce hit lists.  With keep_stored (the checked proof) the kernels
// write StoredHit records and every hit is kept with its bytes (kept()); otherwise the first K2 per nonce (lists()).
// Chunks must be submitted in ascending label order and collected in submission order.
class Scanner {
public:
    ~Scanner() { if (dev_ >= 0) { cudaSetDevice(dev_); drain(); } }   // the members free themselves on the scan's device
    int init(uint32_t provider, const uint8_t challenge[32], uint32_t nonces, const uint64_t *pows, uint32_t k1, uint32_t k2,
             uint64_t num_labels, uint64_t chunk, bool keep_stored = false);
    uint8_t *staging(int b) { return h_labels_[b].get(); }
    // enqueue chunk in staging(b): labels [first, first+count)
    int submit(int b, uint64_t first, uint32_t count);
    // wait for chunk b and fold its hits in.  The fold (hit lists, full nonces, labels scanned) happens under
    // `fold_mu` when given, so that other threads may read that state under the same mutex.
    int collect(int b, std::mutex *fold_mu = nullptr);
    // wait for whatever is still in flight, without folding it (error and cancel paths)
    void drain();
    // start from the hit lists of an earlier scan of the labels below this one's first chunk (at most K2 per nonce)
    void restore(const HitLists &lists);
    const HitLists &lists() const { return lists_; }
    const KeptLists &kept() const { return kept_; }
    KeptLists &kept() { return kept_; }
    bool any_full() const { return full_ > 0; }          // some nonce has K2 hits
    // every nonce has K2 hits (kept: K2 good ones): later labels change no nonce's first K2 (usable) hits
    bool saturated() const { return stored_ ? count_kept(true) == nonces_ : full_ == nonces_; }
    // nonces with at least K2 kept hits (good ones only, or good and pending)
    uint32_t count_kept(bool good_only) const;
    uint32_t nonces() const { return nonces_; }
    uint64_t scanned() const { return scanned_; }
    uint64_t chunk() const { return chunk_; }
    int device() const { return dev_; }
    DeviceEngine *engine() const { return engine_; }

private:
    int fold_stored(int b, uint32_t n, std::mutex *fold_mu);
    template <class Rec>
    void launch(cudaStream_t st, const uint4 *labels, uint64_t first, uint32_t count, Rec *hits, uint32_t *n_hits);

    DeviceEngine *engine_ = nullptr;
    int dev_ = -1;
    uint32_t nonces_ = 0, k2_ = 0, msb_ = 0, hit_cap_ = 0, grid_ = 0, full_ = 0;
    uint64_t lsb_ = 0, chunk_ = 0, scanned_ = 0;
    bool stored_ = false;
    size_t rec_ = 0;   // bytes per hit record (Hit or StoredHit), set by init
    DeviceBuffer<uint8_t> d_rk_, d_lazy_;
    DeviceBuffer<AesTables> d_tables_;
    Stream st_[2];
    Event ev_[2];
    DeviceBuffer<uint8_t> d_labels_[2];
    PinnedBuffer<uint8_t> h_labels_[2];
    DeviceBuffer<uint8_t> d_hits_[2];   // hit_cap_ records of rec_ bytes
    PinnedBuffer<uint8_t> h_hits_[2];
    DeviceBuffer<uint32_t> d_nhits_[2];
    PinnedBuffer<uint32_t> h_nhits_[2], h_ncands_[2];
    DeviceBuffer<uint2> d_cands_;
    DeviceBuffer<uint32_t> d_ncands_;
    uint32_t cand_cap_ = 0;
    bool pending_[2] = {false, false};
    uint32_t count_[2] = {0, 0};
    HitLists lists_;
    KeptLists kept_;
};

extern const char *const kNoProof;   // "no proof found: ..."

// The proof record of winner (nonce, idx): packs the indices, takes the nonce group's pow, counts the proof in the
// metrics with `scanned` labels.
int write_proof(uint64_t scanned, uint32_t nonce, const std::vector<uint64_t> &idx, const uint64_t *pows, uint64_t num_labels,
                b200post_proof_out *out);

// pow_mode and its hook: B200POST_ERR_UNSUPPORTED for an unknown mode or CALLBACK without pow_prove
int check_pow_mode(const b200post_prove_opts &o);
// The k2pow step of a proof: one pow per nonce group for `challenge` under cfg_difficulty / num_units (BUILTIN on
// `providers`, CALLBACK through o.pow_prove, SKIP = 0).  pows gets o.nonces / 16 entries.
int find_pows(const b200post_prove_opts &o, const uint8_t challenge[32], const uint8_t node_id[32], uint32_t num_units,
              const uint8_t cfg_difficulty[32], const uint32_t *providers, int n_providers, std::vector<uint64_t> *pows,
              const volatile int *cancel);
// The verifier gate: the proof through b200post_verify_batch on `provider` (k2pow checked under BUILTIN only).  A
// rejection clears *out and returns B200POST_ERR_INVALID_PROOF with the verifier's reason.
int gate_proof(uint32_t provider, const b200post_post_config &cfg, uint64_t scrypt_n, const b200post_prove_opts &o,
               const b200post_proof_metadata &meta, b200post_proof_out *out);

}  // namespace b200post
