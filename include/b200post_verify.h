/*
 * b200post_verify.h — batched POST proof verification on the GPU label engine (part of libb200post.so).
 *
 * Replaces, for the label-recomputation-heavy part, what go-spacemesh reaches through
 *   activation.PostVerifier            activation/interface.go:26-29
 *   activation.postVerifier.Verify      activation/post_verifier.go:150-160  -> verifying.ProofVerifier.Verify (:159)
 *   activation.offloadingPostVerifier   activation/post_verifier.go:122-142, 230-390 (queue, workers, priorities, Close)
 *   verifying.Subset / SelectedIndex    activation/validation.go:206-209, activation/malfeasance.go:161-166
 *
 * The reference verifies ONE proof per call on NumCPU/2 worker goroutines (activation/post.go:101-111).  Here
 * any number of threads call b200post_verifier_verify() concurrently; a dispatcher drains everything queued
 * (prioritised jobs first), recomputes all requested labels of the batch in one GPU gather and demultiplexes
 * the verdicts.  Semantics kept: safe for concurrent use; "verifier is closed" after Close (B200POST_ERR_CLOSED,
 * activation/post_verifier_test.go:61,90,102); an empty index list is an error (B200POST_ERR_EMPTY_PROOF,
 * activation/e2e/validation_test.go:102); a label that fails the difficulty yields
 * B200POST_ERR_INVALID_PROOF + the POSITION of the offending index in the proof's K2 list (verifying.ErrInvalidIndex{Index}:
 * activation/handler_v1.go:228,248 stores it as InvalidPostIndexProof.InvalidIdx and activation/malfeasance.go:165
 * re-verifies it with verifying.SelectedIndex(InvalidIdx), so it must be a position, also under SUBSET).
 *
 * PARITY NOTE.  Everything outside label recomputation — index bit-packing, the BLAKE3-derived AES-128 keys,
 * the 8/56-bit difficulty compare, Subset(K3, seed) selection — follows the published post-rs v0.7.x
 * behaviour from memory; none of it is pinned by a vector in the reference tree ("parity unpinned",
 * DESIGN.md §2).  The k2pow check is RandomX (cmd/root.go:254-259): by default the verifier computes one RandomX hash
 * per proof on the device (include/b200post_k2pow.h; the RandomX function itself is pinned on its official vectors).
 * A caller-supplied callback or an explicit skip are opt-in (b200post_verifier_opts.pow_mode); a NULL callback no
 * longer means "skip".
 */
#ifndef B200POST_VERIFY_H
#define B200POST_VERIFY_H

#include <stddef.h>
#include <stdint.h>

#include "b200post.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200post_proof {            /* shared.Proof {Nonce, Indices, Pow}  api/grpcserver/post_client.go:124-128 */
    uint32_t nonce;
    const uint8_t *indices;                /* K2 indices, floor(log2(numLabels))+1 bits each, LSB-first bit-packed      */
    size_t indices_len;
    uint64_t pow;
} b200post_proof;

typedef struct b200post_proof_metadata {   /* shared.ProofMetadata  activation/validation.go:193-199 */
    uint8_t node_id[32];
    uint8_t commitment_atx_id[32];
    uint8_t challenge[32];
    uint32_t num_units;
    uint64_t labels_per_unit;
} b200post_proof_metadata;

typedef struct b200post_verify_params {    /* config.Config + ScryptParams  activation/post.go:27-49,59 */
    uint32_t k1, k2;
    uint8_t pow_difficulty[32];
    uint64_t scrypt_n;                     /* r = p = 1 */
} b200post_verify_params;

enum { B200POST_VERIFY_ALL = 0, B200POST_VERIFY_SUBSET = 1, B200POST_VERIFY_SELECTED_INDEX = 2 };

typedef struct b200post_verify_options {
    uint32_t mode;                         /* ALL (K2 indices) | SUBSET (verifying.Subset(k3, seed)) | SELECTED_INDEX */
    uint32_t k3;                           /* SUBSET: how many of the K2 positions to check                           */
    const uint8_t *seed;                   /* SUBSET: selection seed (the local peer ID, activation/handler_v1.go:226) */
    size_t seed_len;
    uint32_t selected_index;               /* SELECTED_INDEX: position (0..K2-1) to check                             */
    uint32_t prioritized;                  /* PrioritizedCall()  activation/interface.go:50-54                          */
} b200post_verify_options;

/* k2pow check hook: return 0 if `pow` is valid.  difficulty = pow_difficulty / num_units (already scaled). */
typedef int (*b200post_pow_verify_fn)(void *ctx, uint64_t pow, uint8_t nonce_group, const uint8_t challenge8[8],
                                      const uint8_t difficulty[32], const uint8_t node_id[32]);

enum { B200POST_POW_BUILTIN = 0, B200POST_POW_CALLBACK = 1, B200POST_POW_SKIP = 2 };

typedef struct b200post_verifier_opts {
    b200post_pow_verify_fn pow_verify;     /* used when pow_mode == B200POST_POW_CALLBACK (must be non-NULL then)        */
    void *pow_ctx;
    uint32_t max_batch_proofs;             /* 0 = 16384; cap on proofs coalesced into one GPU batch                    */
    uint32_t pow_mode;                     /* BUILTIN (default, also with opts == NULL): RandomX on the device;
                                              CALLBACK: pow_verify; SKIP: no k2pow check — must be asked for explicitly  */
    const uint8_t *pow_cache_key;          /* BUILTIN: RandomX cache key, NULL = B200POST_K2POW_DEFAULT_KEY              */
    size_t pow_cache_key_len;
} b200post_verifier_opts;

typedef struct b200post_verifier b200post_verifier;

/* NewPostVerifier (activation/post_verifier.go:191-221).  opts may be NULL (= builtin k2pow check).
 * B200POST_ERR_UNSUPPORTED if pow_mode is CALLBACK without a function. */
int b200post_verifier_new(uint32_t provider, const b200post_verifier_opts *opts, b200post_verifier **out);

/* PostVerifier.Verify: blocking, safe for concurrent use.  options may be NULL (= ALL, not prioritised).
 * Returns B200POST_OK, B200POST_ERR_INVALID_PROOF (*invalid_index = position 0..K2-1 of the failing index in the proof's
 * index list, or UINT64_MAX when the k2pow — not a label — is invalid),
 * B200POST_ERR_EMPTY_PROOF, B200POST_ERR_INVALID_ARGUMENT, B200POST_ERR_CLOSED, or an engine error. */
int b200post_verifier_verify(b200post_verifier *v, const b200post_proof *proof, const b200post_proof_metadata *meta,
                             const b200post_verify_params *params, const b200post_verify_options *options,
                             uint64_t *invalid_index);

/* One dispatcher over several devices: a worker per device drains the same queues (long queues are shared out,
 * short ones go to whichever device is idle).  Verify/Close/free/stats as above. */
int b200post_verifier_new_multi(const uint32_t *providers, int n_providers, const b200post_verifier_opts *opts,
                                b200post_verifier **out);

/* PostVerifier.Close: wakes every waiter with B200POST_ERR_CLOSED; idempotent; later Verify calls fail fast. */
int b200post_verifier_close(b200post_verifier *v);
void b200post_verifier_free(b200post_verifier *v);

/* Proofs coalesced per GPU batch so far: batches dispatched and proofs handled (for tests / metrics). */
int b200post_verifier_stats(b200post_verifier *v, uint64_t *batches, uint64_t *proofs);

/* Synchronous batch form (BASELINE.json configs[2]: 10 000 proofs x K2 = 37): verifies n proofs in one GPU
 * batch on the calling thread.  statuses[i] gets the per-proof code, invalid_indices[i] the failing position. */
int b200post_verify_batch(uint32_t provider, size_t n, const b200post_proof *proofs, const b200post_proof_metadata *metas,
                          const b200post_verify_params *params, const b200post_verify_options *options /* n or NULL */,
                          const b200post_verifier_opts *opts, int *statuses, uint64_t *invalid_indices);

/* The same batch split over `n_providers` devices: contiguous runs of proofs, one host thread per device, no
 * data-path collective (proofs are independent — SURVEY.md §8e).  Results land in the caller's order. */
int b200post_verify_batch_multi(const uint32_t *providers, int n_providers, size_t n, const b200post_proof *proofs,
                                const b200post_proof_metadata *metas, const b200post_verify_params *params,
                                const b200post_verify_options *options /* n or NULL */, const b200post_verifier_opts *opts,
                                int *statuses, uint64_t *invalid_indices);

/* ---------------------------------------------------------------------------------------------------------------
 * VRF-nonce checks in batches.  Validator.VRFNonce / VRFNonceV2 (activation/validation.go:261-285, called by
 * activation/handler_v2.go on every non-initial V2 ATX and by handler_v1.go on initial ATXs) recompute ONE label per
 * check: the label at the nonce.  These calls put many checks into one GPU gather, and the verifier handle coalesces
 * them with concurrent proofs (one gather per scrypt N; the checks' labels follow the proofs' labels).
 *
 * PARITY: *valid / valid[i] is label32 < floor(2^256 / numLabels), strict — the UNPINNED rule of
 * b200post_verify_vrf_nonce, which real network data contradicts as a universal rule (see include/b200post.h).  The
 * label32 at the nonce comes back with it, so that a caller can apply the rule the network uses.
 *
 * A check never reaches the k2pow step, is not counted as a proof (b200post_verifier_stats' proofs, the verify
 * metrics), and counts as one entry toward max_batch_proofs.  Per-check argument errors (num_units * labels_per_unit
 * 0 or above 2^64-1, scrypt N not a power of two in [2, 2^20]) give that check B200POST_ERR_INVALID_ARGUMENT and leave
 * the others alone.  The nonce is not range-checked: a nonce >= numLabels is what the past-the-end search produces.
 * --------------------------------------------------------------------------------------------------------------- */
typedef struct b200post_vrf_check {        /* shared.VRFNonceMetadata + nonce: activation/validation.go:261-285 */
    uint8_t node_id[32];
    uint8_t commitment_atx_id[32];
    uint64_t nonce;
    uint64_t labels_per_unit;
    uint64_t scrypt_n;                     /* r = p = 1 */
    uint32_t num_units;
    uint32_t prioritized;                  /* verifier only: PrioritizedCall */
} b200post_vrf_check;

/* Validator.VRFNonce / VRFNonceV2 through the verifier's dispatcher: blocking, safe for concurrent use, coalesced with
 * concurrent proofs.  B200POST_OK with *valid = label32 < floor(2^256 / numLabels) (the UNPINNED rule of
 * b200post_verify_vrf_nonce), label32 (may be NULL) = the label at the nonce; INVALID_ARGUMENT, CLOSED or an engine error. */
int b200post_verifier_verify_vrf_nonce(b200post_verifier *v, const b200post_vrf_check *c, int *valid, uint8_t label32[32]);

/* n checks in one GPU batch on the calling thread; statuses[i] per item, valid[i] 0/1, labels32 = n x 32 bytes or NULL.
 * Call-level checks, in this order: NULL pointers with n > 0 -> INVALID_ARGUMENT, the CPU provider id -> UNSUPPORTED,
 * no such device -> NO_DEVICE (no fallback), n == 0 -> OK.  A failed item gets valid 0 and a zero label32. */
int b200post_verify_vrf_nonces(uint32_t provider, size_t n, const b200post_vrf_check *checks, int *statuses, int *valid,
                               uint8_t *labels32);
/* the same split over devices: contiguous runs, one host thread each, results in the caller's order */
int b200post_verify_vrf_nonces_multi(const uint32_t *providers, int n_providers, size_t n, const b200post_vrf_check *checks,
                                     int *statuses, int *valid, uint8_t *labels32);

/* Helpers shared with the Go side (all ASSUMED post-rs conventions, see PARITY NOTE). */
uint32_t b200post_bits_per_index(uint64_t num_labels);                       /* floor(log2(num_labels)) + 1       */
uint64_t b200post_proving_difficulty(uint32_t k1, uint64_t num_labels);      /* floor(2^64 * k1 / num_labels)      */
/* pack / unpack `count` indices of `bits` bits each, LSB-first.  Return bytes written / indices read. */
size_t b200post_pack_indices(const uint64_t *indices, size_t count, uint32_t bits, uint8_t *out, size_t out_cap);
size_t b200post_unpack_indices(const uint8_t *packed, size_t packed_len, uint32_t bits, uint64_t *out, size_t out_cap);

#ifdef __cplusplus
}
#endif
#endif /* B200POST_VERIFY_H */
