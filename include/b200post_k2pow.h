/*
 * b200post_k2pow.h — k2pow (RandomX proof of work) on the GPU (part of libb200post.so).
 *
 * What it replaces in the reference (paths relative to spacemeshos/go-spacemesh):
 *   b200post_k2pow_search   -> the k2pow nonce search the external post-service runs before the proving scan, asked for
 *                              by the one blocking RPC at activation/nipost.go:171 (NIPostBuilder.Proof, :114-185);
 *                              result = types.Post.Pow (api/grpcserver/post_client.go:124-128, activation/wire/wire_v1.go:44)
 *   b200post_k2pow_verify   -> the pow check inside verifying.ProofVerifier.Verify (activation/post_verifier.go:150-160,
 *                              external call :159); flags activation/post_types.go:84-121 (PowFlags, RandomXMode)
 *   difficulty              -> PostConfig.PowDifficulty (activation/post.go:27-49, activation/post_types.go:11-38,
 *                              mainnet value config/mainnet.go:41), divided by NumUnits before the compare
 *
 * The function is RandomX (cmd/root.go:254-259): hash = RandomX(cache key, pow[0:7] || nonce_group || challenge[0:8] ||
 * node_id), valid when hash < difficulty as 32 big-endian bytes.  The RandomX arithmetic is pinned on RandomX's own
 * known-answer vectors THROUGH THIS LIBRARY (tests/test_gpu_k2pow.py runs them on the GPU via b200post_randomx_hash);
 * the input layout, the cache key string and the difficulty scaling follow post-rs from memory ("parity unpinned":
 * no k2pow fixture exists in the reference tree).
 *
 * "Fast mode" only: the 2080 MiB dataset is built on the device (once per key and device, ~1 s) and stays in HBM; the
 * reference's light/fast distinction (RandomXMode) is a CPU memory trade-off that an 80 GB device does not need.
 * No CPU fallback: without a CUDA device every call returns B200POST_ERR_NO_DEVICE.
 */
#ifndef B200POST_K2POW_H
#define B200POST_K2POW_H

#include <stddef.h>
#include <stdint.h>

#include "b200post.h"

#ifdef __cplusplus
extern "C" {
#endif

#define B200POST_K2POW_NOT_FOUND UINT64_MAX
#define B200POST_K2POW_DEFAULT_KEY "spacemesh-randomx-cache-key" /* post-rs pow/randomx.rs (recollection) */

typedef struct b200post_k2pow_params {
    const uint8_t *cache_key;      /* NULL = B200POST_K2POW_DEFAULT_KEY */
    size_t cache_key_len;
    uint8_t nonce_group;           /* proving nonce / 16 */
    uint8_t challenge8[8];         /* first 8 bytes of the POST challenge */
    uint8_t node_id[32];
    uint8_t difficulty[32];        /* already divided by num_units (b200post_k2pow_scale_difficulty); big-endian */
} b200post_k2pow_params;

/* pow_difficulty / num_units as 256-bit big-endian integers (post-rs scale_pow_difficulty). */
void b200post_k2pow_scale_difficulty(const uint8_t pow_difficulty[32], uint32_t num_units, uint8_t out[32]);

/* Builds (or finds already resident) the RandomX dataset for `key` on `provider`.  Optional: every other call does it
 * lazily.  key NULL = the default spacemesh key. */
int b200post_randomx_prepare(uint32_t provider, const uint8_t *key, size_t key_len);

/* RandomX hashes of n equally long inputs (HOST buffers: inputs = n x input_len bytes, out32 = n x 32 bytes).
 * Generic entry point: RandomX's published test vectors run through it. */
int b200post_randomx_hash(uint32_t provider, const uint8_t *key, size_t key_len, const uint8_t *inputs, size_t input_len,
                          size_t n, uint8_t *out32);

/* Dataset items [first_item, first_item+count) of `key` on `provider` (out = count x 8 uint64, HOST), building the
 * dataset first if it is not resident.  A range past the 34 078 719 items is INVALID_ARGUMENT.  Diagnostics / tests. */
int b200post_randomx_dataset_read(uint32_t provider, const uint8_t *key, size_t key_len, uint64_t first_item, uint64_t count,
                                  uint64_t *out);

/* k2pow hashes of pow = start .. start+count-1 (out32 = count x 32 bytes, HOST).  Diagnostics / tests. */
int b200post_k2pow_hashes(uint32_t provider, const b200post_k2pow_params *p, uint64_t start, uint64_t count, uint8_t *out32);

/* Nonce search over pow in [start, start+count) (count is clamped to the 56-bit nonce space).  The range is walked in
 * device-sized batches in ascending order; the search stops after the first batch that holds a valid nonce and *found
 * is the smallest one in it (any valid nonce is acceptable to the verifier), else B200POST_K2POW_NOT_FOUND.
 * *hashes_done (may be NULL) = hashes actually computed.  `cancel` (may be NULL) is polled between batches. */
int b200post_k2pow_search(uint32_t provider, const b200post_k2pow_params *p, uint64_t start, uint64_t count,
                          uint64_t *found, uint64_t *hashes_done, const volatile int *cancel);

/* The same range split over several devices (interleaved batches, one host thread per device, no data-path
 * collective: nonces are independent — SURVEY.md §8e).  Stops all devices once any of them has a hit. */
int b200post_k2pow_search_multi(const uint32_t *providers, int n_providers, const b200post_k2pow_params *p,
                                uint64_t start, uint64_t count, uint64_t *found, uint64_t *hashes_done,
                                const volatile int *cancel);

/* What the prover needs (one k2pow per group of 16 proving nonces, activation/post.go:64-81 Nonces): the smallest valid
 * pow of each nonce group 0..n_groups-1 (p->nonce_group is ignored), all groups sharing device batches.  pows[g] =
 * B200POST_K2POW_NOT_FOUND if none below max_nonces_per_group (0 = the whole 56-bit space). */
int b200post_k2pow_search_groups(uint32_t provider, const b200post_k2pow_params *p, uint32_t n_groups, uint64_t max_nonces_per_group,
                                 uint64_t *pows, uint64_t *hashes_done, const volatile int *cancel);

/* The verifier's check: *valid = 1 iff RandomX(input(pow)) < p->difficulty. */
int b200post_k2pow_verify(uint32_t provider, const b200post_k2pow_params *p, uint64_t pow, int *valid);

/* Device time (ms, CUDA events on the engine's stream) and hashes of the most recent k2pow / randomx call on `provider`,
 * and of its VM kernel alone (the dominant kernel).  Any pointer may be NULL. */
int b200post_randomx_last_timing(uint32_t provider, double *total_ms, double *vm_kernel_ms, uint64_t *hashes, uint64_t *vm_launches);

/* VMs (hashes) one device batch holds under the current options ("rx_vm_mode", default 1 = 48 VMs per SM: 6 336 on a
 * 132-SM H100; "rx_vms_per_sm" overrides the count; shrunk to what fits in free HBM at 2 MiB + 16 KiB per VM). */
int b200post_randomx_batch_size(uint32_t provider, uint64_t *vms);

#ifdef __cplusplus
}
#endif
#endif /* B200POST_K2POW_H */
