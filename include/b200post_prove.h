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
    uint64_t labels_scanned;           /* how far the scan had to go                                            */
} b200post_proof_out;

/* Proof over the POST data in `data_dir` (postdata_N.bin + postdata_metadata.json written by a setup session).
 * `meta_out` (optional) receives the matching ProofMetadata.  B200POST_ERR_INVALID_PROOF = the data holds no
 * nonce with K2 qualifying labels ("no proof found"). */
int b200post_generate_proof(const char *data_dir, const uint8_t challenge[32], const b200post_post_config *cfg,
                            const b200post_prove_opts *opts, b200post_proof_out *out, b200post_proof_metadata *meta_out,
                            const volatile int *cancel);

/* The scan alone over labels already in host memory: labels16 = count x 16 bytes holding label indices
 * [first_index, first_index + count).  pows = one u64 per nonce group (nonces/16 of them). */
int b200post_prove_scan(uint32_t provider, const uint8_t *labels16, uint64_t first_index, uint64_t count,
                        const uint8_t challenge[32], uint32_t nonces, const uint64_t *pows, uint32_t k1, uint32_t k2,
                        uint64_t num_labels, b200post_proof_out *out);

#ifdef __cplusplus
}
#endif
#endif /* B200POST_PROVE_H */
