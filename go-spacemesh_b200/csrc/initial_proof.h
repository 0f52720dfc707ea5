// initial_proof.h — the initial POST proof of a full setup session (b200post_setup_request_initial_proof, DESIGN.md §3e):
// the proving scan runs over each label batch as the session writes it, so the first proof needs no second read of
// the data.  The session (setup.cu) drives it; the scan itself is the prover's (prove_internal.h).
// The same class keeps a file-range session's record (b200post_setup_request_range_record, DESIGN.md §3c): the VRF
// best of the range's labels and, optionally, the proving scan of [lo, hi) with no stop rule, which
// b200post_merge_range_records (range_records.cu) merges into the POST's nonce and initial proof.
#pragma once
#include <cstdint>
#include <optional>
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

// A file-range session's files [from_file, to_file] and labels [lo, hi).
struct RangeSpec { uint64_t from_file = 0, to_file = 0, lo = 0, hi = 0; };

// The session's scan of [0, numLabels) with its state file (initial_post.scan), or a range session's record
// (range_<from>_<to>.rec) of [lo, hi).  Calls come from the session's thread in this order: begin, then per batch
// note_vrf (records), buffer + scan (and checkpoint at file ends), then finish (whole POST); stop on cancel or failure.
class InitialProofScan {
public:
    // Before the first label batch: the device check, the state file (pows, scanned prefix, hit lists, and a record's
    // VRF best; ignored unless it is intact, matches and its prefix ends at or below *written), the pows (found and saved
    // when the state gave none; the RandomX engines' HBM is released after a BUILTIN search) and the scanner.
    //   range == nullptr (the whole POST): the gap [upto, *written) is rescanned from the files.
    //   range given (a record): nothing is read back; *written becomes the record's upto, or lo without a usable record,
    //   and the session computes the labels from there.  req == nullptr: the record holds the VRF best only.
    int begin(const InitialProofRequest *req, const RangeSpec *range, const std::string &dir, const b200post_post_metadata &md,
              const b200post_post_config &cfg, int64_t provider_id, uint64_t *written, uint64_t batch, const volatile int *cancel);
    // a record's VRF best so far (found only when below every earlier one: the session's threshold tightens)
    const b200post_vrf_nonce &vrf() const { return vrf_; }
    void note_vrf(const b200post_vrf_nonce &nn) { if (nn.found) vrf_ = nn; }
    // Where the next batch of `count` labels should be computed: a pinned staging buffer of the scanner, or nullptr when
    // the batch is larger than one scan chunk (it is then copied into staging in pieces by scan()).
    int buffer(uint64_t count, uint8_t **dst);
    // labels [first, first + count) at src, the next ones after everything scanned so far
    int scan(uint64_t first, uint64_t count, const uint8_t *src);
    // waits for every scan in flight and saves the state
    int checkpoint();
    // cancel or failure: folds what finished, in order and up to the first failed chunk, then saves the state (best effort)
    void stop();
    // After the last label: the winner (the prover's window decision, ProveRule::decide), the proof record and the
    // verifier gate.  B200POST_ERR_INVALID_PROOF (reason in last_error) when no nonce reached K2 or the gate refused.
    int finish(b200post_proof_out *out, b200post_proof_metadata *meta);

    // A record file read back for the merge: false unless it is intact and laid out as header() writes it.
    bool read_record(const std::string &bytes);
    std::string state_path() const;   // the scan state's or the record's file (a record read back has no directory)
    const b200post_post_metadata &md() const { return md_; }
    const b200post_post_config &cfg() const { return cfg_; }
    const b200post_prove_opts &opts() const { return opts_; }   // pow_cache_key points into this object
    const RangeSpec &range() const { return range_; }
    bool has_proof() const { return proof_; }
    uint32_t windows() const { return windows_; }
    const std::vector<uint64_t> &pows() const { return pows_; }
    const HitBook &hits() { return book(); }
    uint64_t upto() { return proof_ ? range_.lo + book().scanned() : upto_; }   // the end of the covered prefix
    std::string proof_part() const;   // K1, K2, nonces, pow difficulty, pow mode, cache key and W, as in the header

private:
    std::string header() const;
    bool decode(const std::string &s, uint64_t written);
    bool load_state(uint64_t written);
    int save_state();
    int submit_from(const uint8_t *src, uint64_t first, uint64_t count);
    // the scanner's collect / submit, recording the first failure (after it nothing more is folded)
    int collect(int b);
    int submit(int b, uint64_t first, uint64_t count);
    uint32_t nonces() const { return opts_.nonces * windows_; }   // every nonce of the session's windows
    HitBook &book() { return rule_->book(0); }

    bool record_ = false;         // a range session's record, not the whole POST's scan state
    bool proof_ = true;           // the proving scan is part of it (always, for the whole POST)
    RangeSpec range_;             // [0, numLabels) for the whole POST
    b200post_vrf_nonce vrf_{};    // a record's VRF best
    uint64_t upto_ = 0;           // a record without the scan: the end of the labels computed and written
    std::string dir_;
    b200post_prove_opts opts_{};
    uint32_t windows_ = 1;        // nonce windows scanned (the request's windows_per_pass)
    std::vector<uint8_t> key_;
    b200post_post_metadata md_{};
    b200post_post_config cfg_{};
    uint64_t num_labels_ = 0;
    uint32_t scan_dev_ = 0;
    std::vector<uint64_t> pows_;
    std::optional<ProveRule> rule_;   // one shard, unchecked; its book holds the hits of the scanned prefix of [lo, hi)
    Scanner sc_;
    int b_ = 0;                   // staging buffer of the next chunk
    bool failed_ = false;         // a chunk failed to be submitted or collected
};

}  // namespace b200post
