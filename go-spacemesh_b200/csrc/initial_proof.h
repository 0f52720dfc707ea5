// initial_proof.h — the initial POST proof of a full setup session (b200post_setup_request_initial_proof, DESIGN.md §3e):
// the proving scan runs over each label batch as the session writes it, so the first proof needs no second read of
// the data.  The session (setup.cu) drives it; the scan itself is the prover's (prove_internal.h).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/b200post_prove.h"
#include "prove_internal.h"

namespace b200post {

// What b200post_setup_request_initial_proof recorded (the cache key is copied: opts.pow_cache_key points into it).
struct InitialProofRequest {
    b200post_prove_opts opts{};
    std::vector<uint8_t> cache_key;
};

// The session's scan of [0, numLabels) with its state file (initial_post.scan).  Calls come from the session's
// thread in this order: begin, then per batch buffer + scan (and checkpoint at file ends), then finish; stop on
// cancel or failure.
class InitialProofScan {
public:
    // Before the first label batch: the device check, the state file (pows, scanned prefix, hit lists; ignored unless
    // it is intact, matches and its prefix ends at or below `written`), the pows (found and saved when the state gave
    // none; the RandomX engines' HBM is released after a BUILTIN search), the scanner, then the gap [upto, written)
    // rescanned from the files.
    int begin(const InitialProofRequest &req, const std::string &dir, const b200post_post_metadata &md, const b200post_post_config &cfg,
              int64_t provider_id, uint64_t written, uint64_t batch, const volatile int *cancel);
    // Where the next batch of `count` labels should be computed: a pinned staging buffer of the scanner, or nullptr when
    // the batch is larger than one scan chunk (it is then copied into staging in pieces by scan()).
    int buffer(uint64_t count, uint8_t **dst);
    // labels [first, first + count) at src, the next ones after everything scanned so far
    int scan(uint64_t first, uint64_t count, const uint8_t *src);
    // waits for every scan in flight and saves the state
    int checkpoint();
    // cancel or failure: folds what finished, in order and up to the first failed chunk, then saves the state (best effort)
    void stop();
    // After the last label: the winner (pick_winner over the first K2 hits per nonce), the proof record and the
    // verifier gate.  B200POST_ERR_INVALID_PROOF (reason in last_error) when no nonce reached K2 or the gate refused.
    int finish(b200post_proof_out *out, b200post_proof_metadata *meta);

private:
    std::string header() const;
    bool load_state(uint64_t written);
    int save_state();
    int submit_from(const uint8_t *src, uint64_t first, uint64_t count);
    // the scanner's collect / submit, recording the first failure (after it nothing more is folded)
    int collect(int b);
    int submit(int b, uint64_t first, uint64_t count);

    std::string dir_;
    b200post_prove_opts opts_{};
    std::vector<uint8_t> key_;
    b200post_post_metadata md_{};
    b200post_post_config cfg_{};
    uint64_t num_labels_ = 0;
    uint32_t scan_dev_ = 0;
    std::vector<uint64_t> pows_;
    uint64_t start_ = 0;          // where this session's scanner began: the prefix below came from the state file
    HitLists restored_;
    Scanner sc_;
    int b_ = 0;                   // staging buffer of the next chunk
    bool failed_ = false;         // a chunk failed to be submitted or collected
};

extern const char kInitialProofFile[];   // "initial_post.json"
extern const char kInitialScanFile[];    // "initial_post.scan"

}  // namespace b200post
