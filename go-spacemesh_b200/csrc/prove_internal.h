// prove_internal.h — the prover's pieces that the setup session's initial proof (setup.cu, initial_proof.cu) reuses:
// the streaming scan (Scanner: K6a/K6b behind double-buffered pinned staging), the proof record, the no-proof error,
// the k2pow step and the verifier gate.  Defined in prover.cu; the rule they serve is prove_rule.h's.  The scan's
// sidecar check (SumsCheck) serves b200post_generate_proof_sums only.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "../../include/b200post_prove.h"
#include "aes_device.cuh"
#include "engine.h"
#include "label_sums.h"
#include "prove_rule.h"
#include "sums_plan.h"

namespace b200post {

// The sidecar side of one b200post_generate_proof_sums call, shared by its shards and passes: the heal cap, the bad
// digest ranges met (first label -> labels, and whether only the sidecar was wrong), those healed, and the report's sums.
struct SumsCheck {
    struct Bad { uint64_t count; bool sidecar_only; };
    explicit SumsCheck(uint32_t max_heal) : max_heal(max_heal) {}
    const uint32_t max_heal;
    std::mutex mu;                   // guards bad and healed
    std::map<uint64_t, Bad> bad;
    std::set<uint64_t> healed;
    std::atomic<uint64_t> blocks_checked{0}, labels_verified{0}, labels_uncovered{0};
};

// Streaming scan state: device buffers and keys.  It folds each chunk's hits into a hit book.  With keep_stored (the
// checked proof) the kernels write StoredHit records, whose stored bytes go into the book with the hit.
// Chunks must be submitted in ascending label order and collected in submission order.
class Scanner {
public:
    ~Scanner() { if (dev_ >= 0) { cudaSetDevice(dev_); drain(); } }   // the members free themselves on the scan's device
    // Scans the nonces [first_nonce, first_nonce + nonces) (first_nonce a multiple of 16, the end <= 4096); pows[g] is
    // the pow of group first_nonce / 16 + g.  The kernels see pass-relative nonces; the book gets absolute ones.
    int init(uint32_t provider, const uint8_t challenge[32], uint32_t nonces, const uint64_t *pows, uint32_t k1, uint32_t k2,
             uint64_t num_labels, uint64_t chunk, bool keep_stored = false, uint32_t first_nonce = 0);
    uint8_t *staging(int b) { return h_labels_[b].get(); }
    // Proving over checksummed data (keep_stored scans only): every chunk then comes with its plan ranges.  The covered
    // ranges are hashed on the device after the H2D; collect compares their digests with the sidecar's, heals each bad
    // range (its labels recomputed under `commitment` and N into the chunk's device buffer, hashed and scanned again)
    // and folds covered hits as good, the healed range's instead of its stored ones, and uncovered hits as pending.
    // max_ranges: the most ranges a chunk has.
    int use_sums(SumsCheck *sums, const uint8_t commitment[32], uint64_t N, size_t max_ranges, const volatile int *cancel);
    // enqueue chunk in staging(b): labels [first, first+count), made of ranges[0, n_ranges) with sums
    int submit(int b, uint64_t first, uint32_t count, const SumRange *ranges = nullptr, size_t n_ranges = 0);
    // wait for chunk b and fold its hits and its label count into `book`, under `fold_mu` when given, so that other
    // threads may read the book under the same mutex
    int collect(int b, HitBook *book, std::mutex *fold_mu = nullptr);
    // wait for whatever is still in flight, without folding it (error and cancel paths)
    void drain();
    uint64_t chunk() const { return chunk_; }
    int device() const { return dev_; }
    DeviceEngine *engine() const { return engine_; }

private:
    template <class Rec>
    void fold(int b, uint32_t n, HitBook *book, std::mutex *fold_mu);
    template <class Rec>
    void launch(cudaStream_t st, const uint4 *labels, uint64_t first, uint32_t count, Rec *hits, uint32_t *n_hits, uint2 *cands,
                uint32_t cand_cap, uint32_t *n_cands);
    int fold_sums(int b, uint32_t n, HitBook *book, std::mutex *fold_mu);
    int heal(int b, const SumRange &r, const uint8_t stored[32], std::vector<uint8_t> *hits, bool *sidecar_only);

    DeviceEngine *engine_ = nullptr;
    int dev_ = -1;
    uint32_t nonces_ = 0, first_ = 0, msb_ = 0, hit_cap_ = 0, grid_ = 0;
    uint64_t lsb_ = 0, chunk_ = 0;
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
    // use_sums: per buffer the chunk's first label, its ranges, and the range each digest slot belongs to
    SumsCheck *sums_ = nullptr;
    uint8_t commitment_[32] = {0};
    uint64_t N_ = 0;
    const volatile int *cancel_ = nullptr;
    uint64_t first_label_[2] = {0, 0};
    const SumRange *ranges_[2] = {nullptr, nullptr};
    size_t n_ranges_[2] = {0, 0};
    std::vector<size_t> hashed_[2];
    PinnedBuffer<DigestDesc> h_desc_[2];
    DeviceBuffer<DigestDesc> d_desc_[2];
    PinnedBuffer<uint8_t> h_dig_[2];
    DeviceBuffer<uint8_t> d_dig_[2];
    // healing, one range at a time on the chunk's stream, with its own hits and candidate queue (the other chunk may
    // still be in flight); h_heal_n_: hits, candidates
    DeviceBuffer<uint8_t> d_heal_hits_, d_heal_dig_;
    PinnedBuffer<uint8_t> h_heal_hits_, h_heal_dig_;
    DeviceBuffer<uint32_t> d_heal_n_;
    PinnedBuffer<uint32_t> h_heal_n_;
    DeviceBuffer<uint2> d_heal_cands_;
    DeviceBuffer<DigestDesc> d_heal_desc_;
    PinnedBuffer<DigestDesc> h_heal_desc_;
    uint32_t heal_cand_cap_ = 0;
};

// Sets the "no proof found" error of the nonce windows 0 .. windows - 1 of n nonces each; B200POST_ERR_INVALID_PROOF.
int no_proof(uint32_t windows, uint32_t n);

// The proof record of winner (nonce, idx): packs the indices, takes the nonce group's pow (pows[g] is the pow of group
// first_nonce / 16 + g), counts the proof in the metrics with `scanned` labels.
int write_proof(uint64_t scanned, uint32_t nonce, const std::vector<uint64_t> &idx, const uint64_t *pows, uint32_t first_nonce,
                uint64_t num_labels, b200post_proof_out *out);

// pow_mode and its hook: B200POST_ERR_UNSUPPORTED for an unknown mode or CALLBACK without pow_prove
int check_pow_mode(const b200post_prove_opts &o);
// The k2pow step of a proof: one pow per nonce group first_group .. first_group + n_groups - 1 for `challenge` under
// cfg_difficulty / num_units (BUILTIN on `providers`, CALLBACK through o.pow_prove, SKIP = 0).  pows gets n_groups entries.
int find_pows(const b200post_prove_opts &o, const uint8_t challenge[32], const uint8_t node_id[32], uint32_t num_units,
              const uint8_t cfg_difficulty[32], const uint32_t *providers, int n_providers, uint32_t first_group, uint32_t n_groups,
              std::vector<uint64_t> *pows, const volatile int *cancel);
// The verifier gate: the proof through b200post_verify_batch on `provider` (k2pow checked under BUILTIN only).  A
// rejection clears *out and returns B200POST_ERR_INVALID_PROOF with the verifier's reason.
int gate_proof(uint32_t provider, const b200post_post_config &cfg, uint64_t scrypt_n, const b200post_prove_opts &o,
               const b200post_proof_metadata &meta, b200post_proof_out *out);
// The same gate over n proofs of one scrypt N in one b200post_verify_batch call: rcs[i] / errs[i] are proof i's code and
// text (a failure of the call itself is every proof's), and a rejected proof's *outs[i] is cleared.
void gate_proofs(uint32_t provider, const b200post_post_config &cfg, uint64_t scrypt_n, const b200post_prove_opts &o, size_t n,
                 const b200post_proof_metadata *metas, b200post_proof_out *const *outs, int *rcs, std::string *errs);

}  // namespace b200post
