/*
 * b200post_poet.h — PoET registration proof-of-work nonce search on the GPU (SURVEY.md §8f.4).
 *
 * Stands in for `shared.FindSubmitPowNonce(ctx, powChallenge, poetChallenge, nodeID, difficulty)` of the
 * un-vendored github.com/spacemeshos/poet v0.10.4 (go.mod:47), called at activation/poet.go:529-535 when a PoET
 * does not support certificates (a fallback the reference intends to remove, poet.go:517; duration exported as
 * `poet_pow_duration`).  ASSUMED from the published poet sources, "parity unpinned":
 *     hash(nonce) = SHA-256(powChallenge || nodeID || poetChallenge || LE64(nonce))
 *     valid  <=>  hash has at least `difficulty` leading zero bits;  the search returns the LOWEST valid nonce.
 * One SHA-256 compression per candidate (the constant prefix is absorbed into a midstate on the host).
 */
#ifndef B200POST_POET_H
#define B200POST_POET_H

#include <stddef.h>
#include <stdint.h>

#include "b200post.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Searches nonces [start_nonce, start_nonce + max_nonces) in ascending chunks and returns the lowest valid one in
 * *nonce (B200POST_OK), B200POST_ERR_INVALID_PROOF if none exists in the window, B200POST_ERR_CANCELLED when
 * *cancel becomes non-zero.  pow_challenge_len + 32 + poet_challenge_len must be a multiple of 4.
 * *hashes (optional) receives the number of candidates evaluated. */
int b200post_poet_pow_find(uint32_t provider, const uint8_t *pow_challenge, size_t pow_challenge_len,
                           const uint8_t *poet_challenge, size_t poet_challenge_len, const uint8_t node_id[32],
                           uint32_t difficulty, uint64_t start_nonce, uint64_t max_nonces, uint64_t *nonce,
                           uint64_t *hashes, const volatile int *cancel);

/* The hash itself (host, one candidate), for verification by callers and tests. */
void b200post_poet_pow_hash(const uint8_t *pow_challenge, size_t pow_challenge_len, const uint8_t *poet_challenge,
                            size_t poet_challenge_len, const uint8_t node_id[32], uint64_t nonce, uint8_t out[32]);

#ifdef __cplusplus
}
#endif
#endif /* B200POST_POET_H */
