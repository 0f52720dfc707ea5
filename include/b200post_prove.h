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
 * The k2pow itself is RandomX (cmd/root.go:254-259) and is NOT implemented: `pow_prove` supplies the pow of a
 * nonce group (e.g. libpost's prover); NULL uses pow = 0, which only a verifier without a pow check accepts.
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
} b200post_prove_opts;

typedef struct b200post_proof_out {    /* types.Post / shared.Proof */
    uint32_t nonce;
    uint64_t pow;
    size_t indices_len;
    uint8_t indices[800];              /* wire cap, activation/wire/wire_v1.go:43                               */
    uint64_t labels_scanned;           /* labels streamed from the first index, in whole chunks (not an absolute
                                          index): last proof index - first index < labels_scanned <= labels
                                          offered (count, or num_labels for b200post_generate_proof)           */
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

/*
 * The initial proof of a POST, produced by its setup session (DESIGN.md §3e).  go-spacemesh asks for it right after
 * initialisation (BuildInitialPost: PostClient.Proof(ctx, nodeID, shared.ZeroChallenge, nil)); a proof over 32 zero bytes
 * computed from the labels as the session writes them spares that second read of every stored label.
 *
 * b200post_setup_request_initial_proof: between prepare and start of a session over the whole POST (a file-range session:
 * B200POST_ERR_STATE; not prepared: B200POST_ERR_STATE); prepare clears the request, a second call replaces it.  From
 * opts: nonces (0 = 16; else a positive multiple of 16, <= 4096, or INVALID_ARGUMENT), pow_mode with pow_prove/pow_ctx
 * (CALLBACK without a function: UNSUPPORTED) and the RandomX cache key (copied); provider and chunk_labels are ignored.
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
/* After the session is COMPLETE: its initial proof and ProofMetadata (meta may be NULL), or INVALID_PROOF with the reason.
 * Before that, or when the session did not ask for one: B200POST_ERR_STATE. */
int b200post_setup_initial_proof(b200post_setup_manager *mgr, b200post_proof_out *out, b200post_proof_metadata *meta);
/* The post-service side: the proof in data_dir/initial_post.json, without a scan, if it was made for this POST's
 * metadata (identity, NumUnits, LabelsPerUnit), cfg (LabelsPerUnit, K1, K2, pow difficulty) and `nonces` (0 = 16), for
 * the zero challenge.  Absent, unreadable or stale: B200POST_ERR_IO, "no initial proof: ..."; the caller then proves from
 * the stored data (b200post_generate_proof_checked).  meta may be NULL. */
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
