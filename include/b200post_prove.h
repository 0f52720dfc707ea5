/*
 * b200post_prove.h — POST proof generation scan on the GPU (part of libb200post.so).  SURVEY.md §8f.3.
 *
 * What it stands in for: the AES scan half of `PostClient.Proof` (activation/interface.go:204-207), which in
 * the reference is one blocking RPC (activation/nipost.go:171, api/grpcserver/post_client.go:69-143) into the
 * external post-service (post-rs): after the k2pow search it streams every stored 16-byte label through
 * `Nonces/16` AES-128 ciphers and collects, per nonce, the indices whose ciphertext byte is below the proving
 * difficulty until one nonce has K2 of them (PostProvingOpts{Threads, Nonces}, activation/post.go:64-81;
 * mainnet Nonces = 288, config/mainnet.go:60-65).  Result = types.Post{Nonce, Indices, Pow}
 * (post_client.go:124-128), exactly what b200post_verifier_verify consumes.
 *
 * The k2pow is RandomX (cmd/root.go:254-259): pow_mode BUILTIN (the default) searches it on the device
 * (b200post_k2pow.h); CALLBACK takes it from `pow_prove` (e.g. libpost's prover); SKIP uses pow = 0, which only a
 * verifier without a pow check accepts.
 * All conventions are the post-rs Prover8_56 ones from memory: ASSUMED, "parity unpinned" (DESIGN.md §2).
 * Selection rule (deterministic): among nonces that reach K2 hits, the one whose K2-th hit has the lowest
 * label index wins; ties go to the lower nonce; its first K2 hit indices, ascending, are the proof.
 */
#ifndef B200POST_PROVE_H
#define B200POST_PROVE_H

#include <stddef.h>
#include <stdint.h>

#include "b200post_setup.h"
#include "b200post_verify.h"

#ifdef __cplusplus
extern "C" {
#endif

/* k2pow hook: find `*pow` for (nonce_group, challenge[0:8], node_id) under `difficulty` (already scaled by
 * num_units).  Return 0 on success. */
typedef int (*b200post_pow_prove_fn)(void *ctx, uint8_t nonce_group, const uint8_t challenge8[8],
                                     const uint8_t difficulty[32], const uint8_t node_id[32], uint64_t *pow);

typedef struct b200post_prove_opts {
    uint32_t provider;                 /* CUDA ordinal                                                         */
    uint32_t nonces;                   /* PostProvingOpts.Nonces: a positive multiple of 16 (0 = 16), <= 4096  */
    uint64_t chunk_labels;             /* labels per H2D chunk (0 = 2^22 = 64 MiB)                             */
    b200post_pow_prove_fn pow_prove;   /* used when pow_mode == B200POST_POW_CALLBACK                            */
    void *pow_ctx;
    uint32_t pow_mode;                 /* B200POST_POW_BUILTIN (default): k2pow search on the device (b200post_k2pow.h);
                                          B200POST_POW_CALLBACK: pow_prove; B200POST_POW_SKIP: pow = 0 for every group
                                          (explicit opt-out: such a proof only verifies with the pow check skipped)  */
    const uint8_t *pow_cache_key;      /* BUILTIN: RandomX cache key, NULL = the spacemesh default                 */
    size_t pow_cache_key_len;
    uint32_t max_windows;              /* nonce windows to try (see "Nonce windows" below): 0 or 1 = [0, nonces)
                                          only; B200POST_PROVE_ALL_WINDOWS = up to the group limit (libpost's loop);
                                          any value is clamped to floor(4096 / nonces)                          */
    uint32_t windows_per_pass;         /* windows scanned per read of the POST: 0 or 1 = one; clamped to the
                                          windows left                                                            */
} b200post_prove_opts;

#define B200POST_PROVE_ALL_WINDOWS UINT32_MAX

/* Nonce windows.  With n = nonces, window w is the nonces [w*n, (w+1)*n), nonce groups w*n/16 .. (w+1)*n/16 - 1; only
 * whole windows below nonce 4096 exist (the group is one byte of the k2pow input), so at most floor(4096 / n).  The
 * proof comes from the lowest window in which some nonce reaches K2 (usable, for the checked call) hits; inside it the
 * selection rule above applies and the pow is that nonce group's.
 * A pass scans windows [a, a + m) in one read of the data (m = windows_per_pass): the pows of all m*n/16 groups first,
 * then the scan, which stops early only once window a is decided (the usual stop rule restricted to window a's
 * nonces), or when a shard is saturated for every nonce of the pass; otherwise it reads every label.  The lowest window
 * of the pass with a winner gives the proof; with none, the next pass starts at window a + m.  So the proof does not
 * depend on windows_per_pass, the device list or the chunk size: it is the one sequential windows give, and a pass
 * never reads more labels than they would (it may only find pows for windows that turn out not to be needed).
 * No window up to max_windows with a proof: B200POST_ERR_INVALID_PROOF, "no proof found: ..." naming the windows. */

typedef struct b200post_proof_out {    /* types.Post / shared.Proof */
    uint32_t nonce;
    uint64_t pow;
    size_t indices_len;
    uint8_t indices[800];              /* wire cap, activation/wire/wire_v1.go:43                               */
    uint64_t labels_scanned;           /* labels streamed from the first index, in whole chunks (not an absolute
                                          index), summed over the passes of a windowed proof (so it may exceed
                                          num_labels): in the last pass, last proof index - first index <
                                          its labels <= labels offered (count, or num_labels for the generators) */
} b200post_proof_out;

/* Proof over the POST data in `data_dir` (postdata_N.bin + postdata_metadata.json written by a setup session).
 * `meta_out` (optional) receives the matching ProofMetadata.  B200POST_ERR_INVALID_PROOF = the data holds no
 * nonce with K2 qualifying labels ("no proof found"). */
int b200post_generate_proof(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg,
                            const b200post_prove_opts *opts, b200post_proof_out *out, b200post_proof_metadata *meta_out,
                            const volatile int *cancel);

/* The same proof on several devices (b200post_generate_proof is its one-provider case).  opts->provider is ignored;
 * `providers` (n_providers >= 1 entries, repeats allowed: such shards share the device) takes its place.
 *   k2pow (BUILTIN): b200post_k2pow_search_groups_multi over the same list.  CALLBACK and SKIP as for one device.
 *   scan: [0, numLabels) is split into contiguous shards of whole chunks, one per list entry in list order, sized
 *         within one chunk of each other (a shard may be empty); each shard runs on its own host thread with its own
 *         buffers and reader and keeps, per nonce, its first K2 hits.  The lists merge in shard order (first K2 kept)
 *         and the one-device selection rule picks the winner, so (nonce, indices, pow) are byte-identical to one
 *         device's for the same inputs, chunk size and pows.
 *   stop: once the hits below the end of the gap-free scanned prefix give a nonce K2 of them, every shard stops; a
 *         shard also stops once every nonce has K2 hits inside it.
 *   labels_scanned = the sum over shards (the metric grows by the same); `cancel` is polled per chunk in every shard.
 * Errors: arguments, then metadata (B200POST_ERR_IO), then B200POST_ERR_NO_DEVICE / UNSUPPORTED (CPU id), as for one
 * device.  A read or device error in ANY shard fails the call once every thread has joined (the first failing shard in
 * list order gives the status and text).  Unlike one device, a shard can reach damaged or missing data past the point
 * where a one-device scan would already have stopped with a proof. */
int b200post_generate_proof_multi(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg,
                                  const b200post_prove_opts *opts, const uint32_t *providers, int n_providers,
                                  b200post_proof_out *out, b200post_proof_metadata *meta_out, const volatile int *cancel);

/* What b200post_generate_proof_checked found while proving. */
typedef struct b200post_prove_check {
    uint64_t labels_rechecked;         /* scan hits recomputed and compared with their stored bytes              */
    uint64_t damaged;                  /* distinct label indices among them whose stored bytes differ: damage    */
    uint32_t n_reported;
    uint64_t damaged_index[64];        /* the lowest n_reported damaged label indices, ascending                  */
    uint32_t proof_verified;           /* 1: the returned proof passed b200post_verify_batch                     */
    uint32_t rounds;                   /* recheck rounds run                                                      */
} b200post_prove_check;

/* b200post_generate_proof_multi over stored data that may be damaged (bit rot, a bad drive, a truncated copy).
 * A stored label counts as a hit of a nonce only when it passes the nonce's difficulty AND equals the label recomputed
 * from blake3(NodeId || CommitmentAtxId) at its index under the metadata's scrypt N.  The proof is the one-device
 * selection rule applied to those usable hits, so it depends on the stored data and the real labels only, not on the
 * device list or the chunk size; on undamaged data (nonce, indices, pow) are byte-identical to
 * b200post_generate_proof_multi's.
 *   How: the scan keeps every hit with its 16 stored bytes.  Whenever the multi-device stop rule would fire, the
 *   tentative winner (over unrejected hits below the end of the gap-free scanned prefix) has its not yet rechecked hits
 *   among its first K2 recomputed on the device (K2s/K2p + K3c, the verify_pos path); damaged hits are dropped and the
 *   decision is taken again.  The scan stops only when the winner's first K2 hits are all rechecked.  A shard's own
 *   saturation stop likewise needs K2 rechecked hits for every nonce.
 *   Gate: before returning, the proof goes through b200post_verify_batch on providers[0] (k2pow checked under
 *   pow_mode BUILTIN, not under SKIP or CALLBACK); a rejection returns B200POST_ERR_INVALID_PROOF and no proof.
 *   check: labels_rechecked, the damage found and the lowest 64 damaged indices.  The report is a LOWER BOUND on the
 *   damage and may differ between device lists and chunk sizes; it never names an undamaged label, and it names every
 *   damaged hit among the first K2 hits of every nonce that was ever the tentative winner.  Not seen: a damaged label
 *   that falsely FAILS the difficulty (never a hit; harmless to the proof) and damage past the decision point.  The
 *   full check of the stored data is b200postcli -verify -fraction 100 (b200post_verify_pos).
 * Damage alone is not an error: B200POST_OK with a valid proof and a non-zero report.  Arguments (check NULL included),
 * host checks and their order, cancellation and read errors are those of b200post_generate_proof_multi; metadata with
 * an invalid scrypt N is B200POST_ERR_IO.  A one-device call is a list of one. */
int b200post_generate_proof_checked(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg,
                                    const b200post_prove_opts *opts, const uint32_t *providers, int n_providers,
                                    b200post_proof_out *out, b200post_proof_metadata *meta_out, b200post_prove_check *check,
                                    const volatile int *cancel);

/* Options of b200post_generate_proof_sums (NULL = the defaults). */
typedef struct b200post_prove_sums_opts {
    uint32_t max_heal_blocks;          /* bad blocks the call may recompute; 0 = 1024 (1 GiB of labels)             */
} b200post_prove_sums_opts;

/* What b200post_generate_proof_sums found in the POST's block checksums (postdata_N.sum, b200post_setup.h). */
typedef struct b200post_prove_sums_report {
    uint64_t blocks_checked;           /* digest ranges read, hashed and compared (summed over passes)             */
    uint64_t labels_verified;          /* labels in ranges whose digest matched (summed over passes)               */
    uint64_t labels_uncovered;         /* labels read with no usable sidecar: the checked rule (summed over passes) */
    uint64_t bad_blocks;               /* distinct ranges whose stored digest differed                             */
    uint64_t healed_blocks;            /* distinct bad ranges recomputed and scanned from the recomputation        */
    uint64_t sidecar_only;             /* of the bad ranges: the stored bytes were right, the digest wrong          */
    uint32_t n_reported, reserved;
    b200post_sums_block bad[64];       /* the lowest n_reported bad ranges, ascending                               */
} b200post_prove_sums_report;

/* b200post_generate_proof_checked with the POST's block checksums in the loop: each epoch's proof read becomes a check
 * of every covered label it reads, at no extra read (DESIGN.md §5, "Proving over checksummed data").
 *   Coverage: a label is covered when a usable sidecar of its file (what b200post_check_sums accepts) describes it.  A
 *   digest range is one sidecar digest's labels: 2^16 aligned to the file's first label, or the short last range up to
 *   `covered`.  The scan reads whole ranges per chunk (chunk_labels is an upper bound, raised to 2^16), hashes each
 *   covered range on the device and compares it with its digest.
 *     digest matches: every hit in the range is usable at once (sidecars are only made from device-computed labels).
 *     digest differs (a bad block): the range is recomputed on the scan's device under the metadata's N, hashed again
 *       and scanned from the recomputation; the stored bytes' hits there are discarded.  The recomputed digest equals
 *       the stored one: only the sidecar is wrong (sidecar_only); it equals the sidecar's: the data is damaged.
 *     uncovered (past `covered`, or a file without a usable sidecar): the checked call's rule, hits rechecked.
 *   The proof is the selection rule over those usable hits, with the checked call's stop rule, windows, shards and
 *   verifier gate.  So when every label read is covered, (nonce, indices, pow) are byte-identical to
 *   b200post_generate_proof_multi's over the undamaged POST whatever the damage, device list, chunk size or windows;
 *   without any usable sidecar they and the status are b200post_generate_proof_checked's.  On clean covered data
 *   check->labels_rechecked is 0.
 *   Read-only: the call writes nothing into data_dir; repair stays b200post_check_sums with repair = 1.
 *   Heal cap: more than sopts->max_heal_blocks distinct bad ranges met returns B200POST_ERR_LABEL_MISMATCH ("more than
 *   M damaged blocks: repair first") with `sums` filled and no proof.  As with a read error, a shard can meet bad blocks
 *   past the point where one device would already have stopped, so a device list can reach the cap where one device
 *   does not.
 * Errors and their order are the checked call's (arguments, `sums` NULL included; metadata and an invalid scrypt N:
 * B200POST_ERR_IO; pow mode; NO_DEVICE / UNSUPPORTED for the CPU id; CANCELLED).  A missing or unusable sidecar is
 * never an error.  check and sums are cleared past the argument checks; sums is filled whatever the outcome. */
int b200post_generate_proof_sums(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg,
                                 const b200post_prove_opts *opts, const uint32_t *providers, int n_providers,
                                 const b200post_prove_sums_opts *sopts, b200post_proof_out *out, b200post_proof_metadata *meta_out,
                                 b200post_prove_check *check, b200post_prove_sums_report *sums, const volatile int *cancel);

/* One identity's proof in b200post_generate_proofs. */
typedef struct b200post_prove_item {
    const char *data_dir;              /* in                                                                          */
    uint8_t challenge[32];             /* in: per identity (identities registered at different PoETs differ)          */
    int32_t status;                    /* out: what the one-identity call returns for this item                       */
    char error[256];                   /* out: that call's b200post_last_error() text (truncated), "" when OK         */
    b200post_proof_out proof;          /* out: valid when status is OK                                                */
    b200post_proof_metadata meta;      /* out: valid when status is OK                                                */
    b200post_prove_check check;        /* out: filled when `checked`                                                  */
} b200post_prove_item;

/* Proofs of several identities' POSTs in one call (a node that proves for several identities at once, DESIGN.md §5).
 * Contract: for every item, (nonce, indices, pow), labels_scanned, the check report and status equal those of
 * b200post_generate_proof_checked (checked = 1) or b200post_generate_proof_multi (checked = 0) called for that item
 * alone with the same opts and provider list, whatever the other items, their order and parallel_scans.
 *   k2pow (BUILTIN): the pows of the current pass of every item still proving go into ONE b200post_k2pow_search_jobs
 *     search over `providers`, so identities share device batches.  CALLBACK and SKIP behave per item as in the single call.
 *   scans: an item's scan (the single call's, over `providers`) starts as soon as all of its pass's pows are final,
 *     while the search goes on for the others; at most parallel_scans scans run at once (0 = min(n, 4)), which bounds
 *     pinned staging at parallel_scans x n_providers x 2 x chunk_labels x 16 bytes.  An item that needs another pass
 *     (max_windows) joins the next search.
 *   gate (checked): the proofs go through b200post_verify_batch on providers[0] together, one call per scrypt N among
 *     them, instead of one call each.
 * Errors: an item's failure stays with that item (missing or corrupt metadata, a read error, "no proof found", a gate
 * rejection, a device error of its scan or search).  The call itself returns, in the single call's order:
 * B200POST_ERR_INVALID_ARGUMENT for bad call arguments (items NULL, n 0, cfg NULL, no providers, an item without
 * data_dir; no item is touched), B200POST_ERR_UNSUPPORTED for opts' pow mode, B200POST_ERR_NO_DEVICE / UNSUPPORTED
 * for the device list (checked once some item passed its host checks; those items get the same code and text), and
 * B200POST_ERR_CANCELLED when `cancel` stopped any item (those items report CANCELLED and no proof); else B200POST_OK. */
int b200post_generate_proofs(b200post_prove_item *items, size_t n, const b200post_post_config *cfg,
                             const b200post_prove_opts *opts, const uint32_t *providers, int n_providers,
                             uint32_t checked, uint32_t parallel_scans, const volatile int *cancel);

/*
 * The initial proof of a POST, produced by its setup session (DESIGN.md §3e).  go-spacemesh asks for it right after
 * initialisation (BuildInitialPost: PostClient.Proof(ctx, nodeID, shared.ZeroChallenge, nil)); a proof over 32 zero bytes
 * computed from the labels as the session writes them spares that second read of every stored label.
 *
 * b200post_setup_request_initial_proof: between prepare and start of a session over the whole POST (a file-range session:
 * B200POST_ERR_STATE, it asks for a range record instead, see below; not prepared: B200POST_ERR_STATE); prepare clears the request, a second call replaces it.  From
 * opts: nonces (0 = 16; else a positive multiple of 16, <= 4096, or INVALID_ARGUMENT), pow_mode with pow_prove/pow_ctx
 * (CALLBACK without a function: UNSUPPORTED), the RandomX cache key (copied) and windows_per_pass, the W nonce windows the
 * session scans in its single pass (0 = 1, clamped to floor(4096 / nonces)); provider, chunk_labels and max_windows are
 * ignored.  The proof is then b200post_generate_proof's with the same nonces and max_windows = W; initial_post.json gets
 * a "Windows": W field and initial_post.scan's header ends with W, both only for W > 1 (one-window files are unchanged).
 * K1, K2 and the pow difficulty are the manager's b200post_post_config.
 * The session then (1) finds one pow per nonce group for the zero challenge before its first label batch (BUILTIN on the
 * session's devices, then their RandomX memory is released so that the label layer keeps its size), (2) runs the
 * proving scan (K6a/K6b on the first device of the session) over each batch of [0, numLabels) as it is written, with no
 * stop rule, keeping each nonce's first K2 hits, and (3) once every label is on disk and the VRF nonce is settled, picks
 * the winner with the prover's rule, passes the proof through b200post_verify_batch (k2pow checked under BUILTIN only) and
 * writes it to initial_post.json in the data dir (tmp + rename).  (nonce, indices, pow) are byte-identical to
 * b200post_generate_proof's over the written files with the same config, nonces and pows; labels_scanned = numLabels.
 * Stop and resume: initial_post.scan (the pows, the end of the scanned prefix and the hit lists, checksummed) is saved at
 * every completed postdata file and whenever the session stops or fails.  On start, a state that is missing, damaged,
 * made for other inputs or ahead of the data on disk is ignored; whatever is on disk past the state is rescanned from
 * the files before the session continues.  b200post_setup_reset deletes both files.
 * No nonce with K2 hits, or a proof the gate refuses: the session still completes (its job is the labels), no proof
 * file is written and b200post_setup_initial_proof returns B200POST_ERR_INVALID_PROOF with the reason.  Without a GPU,
 * start_session returns B200POST_ERR_NO_DEVICE (no CPU path) and writes no state.
 */
int b200post_setup_request_initial_proof(b200post_setup_manager *mgr, const b200post_prove_opts *opts);
/*
 * One POST initialised on several machines (DESIGN.md §3c, §3e): each file-range session keeps a record of what its
 * labels contribute, and b200post_merge_range_records turns the records into the POST's VRF nonce and initial proof
 * without reading a stored label.
 *
 * b200post_setup_request_range_record: between b200post_setup_prepare_files and start, for a range short of the whole
 * POST whose metadata has no nonce (not prepared, a whole-POST session or metadata with a nonce: B200POST_ERR_STATE).
 * proof == NULL: the record holds the VRF candidate only.  Otherwise also the initial-proof scan, with the fields of
 * b200post_setup_request_initial_proof (nonces, pow_mode/pow_prove/pow_ctx, the cache key (copied), windows_per_pass)
 * and its errors (bad nonces: INVALID_ARGUMENT; CALLBACK without a function: UNSUPPORTED).  Prepare clears the request,
 * a second call replaces it.
 * The session then computes every batch with the VRF scan on, from the threshold floor(2^256 / numLabels) of the whole
 * POST, tightened to the best label found so far; the best (found, index, label32) goes into the record, not into the
 * metadata, which keeps VrfScanPending and no nonce.  With proof, the pows of the zero challenge for all groups of the
 * W windows are found first (then the RandomX memory is released), and each batch goes through the proving scan as it is
 * written, over [lo, hi), with no stop rule: each nonce keeps its first K2 hits in the range.
 * The record is range_<from>_<to>.rec in the data dir (tmp + rename, FNV-1a 64 checksum): a header with everything its
 * result depends on (identity, NumUnits, LabelsPerUnit, MaxFileSize, scrypt N, the files and labels [lo, hi), and for
 * the proof K1, K2, nonces, W, pow difficulty, pow mode and cache key), then upto (the end of the covered prefix), the
 * VRF best, and for the proof the pows and hit lists.  It is saved at every completed postdata file, when the session
 * stops or fails, and at the end (upto == hi).
 * Resume: a record that is intact, matches and has upto at or below the labels on disk is used, and the session resumes
 * at upto, computing [upto, written) again over the same bytes; any other record is ignored and the range is computed
 * from lo.  A record so speaks only of computed labels, never of stored bytes.  The status counts from the resume point.
 * b200post_setup_reset deletes range_*.rec and their .tmp files.  Without a request a range session writes no record.
 */
int b200post_setup_request_range_record(b200post_setup_manager *mgr, const b200post_prove_opts *proof);

typedef struct b200post_merge_opts {
    int64_t provider_id;               /* CUDA ordinal or B200POST_PROVIDER_ALL: the past-the-end search and the gate   */
    uint64_t compute_batch_size;       /* past-the-end batch, 0 = 2^20 (the init's batch gives the init's LastPosition) */
} b200post_merge_opts;

typedef struct b200post_merge_result {
    uint32_t ranges;                   /* records merged                                                              */
    b200post_vrf_nonce nonce;          /* what the metadata now holds                                                 */
    uint32_t past_end;                 /* 1: no label below the threshold; the past-the-end search found it          */
    int32_t proof_rc;                  /* OK: initial_post.json written; INVALID_PROOF: no nonce reached K2 or the
                                          gate refused; STATE: the records hold no common proof scan                  */
    char proof_reason[256];
    b200post_proof_out proof;
} b200post_merge_result;

/* Merges the range records in data_dir (every postdata file and one range's metadata copied in beside them).
 * Host checks first, before any device is touched; each refusal leaves the metadata and initial_post.json untouched:
 * metadata present (B200POST_ERR_IO); every range_*.rec intact (B200POST_ERR_IO naming the file) and made for this
 * metadata (B200POST_ERR_CONFIG_MISMATCH); the records tile [0, numLabels) with no gap or overlap and each is complete
 * (B200POST_ERR_STATE naming the uncovered labels or the record); every postdata file present with its implied size
 * (B200POST_ERR_IO, "POST data is incomplete"); then B200POST_ERR_UNSUPPORTED for the CPU id and NO_DEVICE without a GPU.
 * Nonce: the minimum of the records' VRF bests under (label32, index), then the rule of an init (below the threshold:
 * LastPosition 0; else the past-the-end search on provider_id, resumable); VrfScanPending is cleared and the metadata
 * saved.  No stored label is read.
 * Initial proof, once the nonce is settled: every record must carry the proof part with the same K1, K2, nonces, W, pow
 * difficulty (also cfg's), pow mode and cache key, and the same pows; the records' hit lists go into the prover's rule as
 * one shard each in range order, the winner goes through the verifier gate on the first device of provider_id and into
 * initial_post.json.  Without a proof, any initial_post.json in data_dir is deleted.  The nonce fields and
 * initial_post.json are byte-identical to those of one uninterrupted full session with the initial proof.
 * Returns OK once the nonce is settled (proof_rc says what became of the proof), CANCELLED when stopped. */
int b200post_merge_range_records(const char *data_dir, const b200post_post_config *cfg, const b200post_merge_opts *o,
                                 b200post_merge_result *out, const volatile int *cancel);

/* After the session is COMPLETE: its initial proof and ProofMetadata (meta may be NULL), or INVALID_PROOF with the reason.
 * Before that, or when the session did not ask for one: B200POST_ERR_STATE. */
int b200post_setup_initial_proof(b200post_setup_manager *mgr, b200post_proof_out *out, b200post_proof_metadata *meta);
/* The post-service side: the proof in data_dir/initial_post.json, without a scan, if it was made for this POST's
 * metadata (identity, NumUnits, LabelsPerUnit), cfg (LabelsPerUnit, K1, K2, pow difficulty) and `nonces` (0 = 16), for
 * the zero challenge.  A file with "Windows": W may hold any nonce below nonces x W.  Absent, unreadable or stale:
 * B200POST_ERR_IO, "no initial proof: ..."; the caller then proves from the stored data (b200post_generate_proof_checked).
 * meta may be NULL. */
int b200post_load_initial_proof(const char *data_dir, const b200post_post_config *cfg, uint32_t nonces, b200post_proof_out *out,
                                b200post_proof_metadata *meta);

/* The scan alone over labels already in host memory: labels16 = count x 16 bytes holding label indices
 * [first_index, first_index + count).  pows = one u64 per nonce group (nonces/16 of them). */
int b200post_prove_scan(uint32_t provider, const uint8_t *labels16, uint64_t first_index, uint64_t count,
                        const uint8_t challenge[32], uint32_t nonces, const uint64_t *pows, uint32_t k1, uint32_t k2,
                        uint64_t num_labels, b200post_proof_out *out);

#ifdef __cplusplus
}
#endif
#endif /* B200POST_PROVE_H */
