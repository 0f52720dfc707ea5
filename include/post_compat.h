/*
 * post_compat.h — the subset of libpost's C header (`post.h`, post-rs v0.7.13) that the POST *label*
 * path of github.com/spacemeshos/post v0.12.9 binds through cgo, re-declared so that libb200post.so can
 * stand in for `-lpost` on that path (link mechanics: Makefile-libs.Inc:5-6,59-69 in the reference;
 * call sites: activation/post.go:295,355-361, activation/post_supervisor.go:106,121).
 *
 * `post.h` is NOT present in the go-spacemesh tree (it is fetched at build time, Makefile-libs.Inc:78-94),
 * so these declarations are a restatement of the published header and are marked "unpinned" in
 * DESIGN.md: a maintainer must diff them against the real post.h before linking.
 *
 * Semantics kept from libpost:
 *   - `initialize(init, start, end, out, &nonce)`: `end` is INCLUSIVE; `out` receives 16 bytes per label;
 *     returns InitializeOk when a VRF nonce below the (running) difficulty was found in this range and
 *     stores its index in *nonce, else InitializeOkNonceNotFound.
 *   - the callee never frees or retains caller memory; an Initializer is used by one thread at a time.
 * Difference: provider id 0xffffffff (CPU) is refused — this library has no CPU path by design.
 */
#ifndef B200POST_POST_COMPAT_H
#define B200POST_POST_COMPAT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum DeviceClass { DeviceClassCPU = 1, DeviceClassGPU = 2 } DeviceClass;

typedef struct Provider {
    char name[64];
    uint32_t id;
    DeviceClass class_;
} Provider;

typedef enum DeviceInfoResult {
    DeviceInfoOk = 0,
    DeviceInfoInvalidArgument = 1,
    DeviceInfoBufferTooSmall = 2,
    DeviceInfoFailed = 3
} DeviceInfoResult;

typedef enum InitializeResult {
    InitializeOk = 0,
    InitializeOkNonceNotFound = 1,
    InitializeInvalidLabelsRange = 2,
    InitializeError = 3,
    InitializeInvalidArgument = 4
} InitializeResult;

typedef struct Initializer Initializer;

size_t get_providers_count(void);
DeviceInfoResult get_providers(Provider *out, size_t out_len);

/* n = scrypt N; commitment = 32 bytes; vrf_difficulty = 32 bytes big-endian or NULL. NULL on error. */
Initializer *new_initializer(uint32_t provider_id, size_t n, const uint8_t *commitment, const uint8_t *vrf_difficulty);
InitializeResult initialize(Initializer *init, uint64_t start, uint64_t end, uint8_t *out, uint64_t *nonce);
void free_initializer(Initializer *init);

/* ---- verifying / proving half of post.h (what verifying.ProofVerifier and the post-service bind) ---------------------
 * Restated from memory of post-rs v0.7.x ffi (post_impl.rs); same "unpinned" caveat as above.  These are what make
 * libb200post.so linkable in place of -lpost for the whole cgo package github.com/spacemeshos/post/internal/postrs
 * (activation/post_verifier.go:159,204; link mechanics Makefile-libs.Inc:5-6,59-69). */
typedef struct ArrayU8 { uint8_t *ptr; size_t len; size_t cap; } ArrayU8;
typedef struct Proof { uint32_t nonce; ArrayU8 indices; uint64_t pow; } Proof;               /* shared.Proof */
typedef struct ProofMetadata {                                                                 /* shared.ProofMetadata */
    uint8_t node_id[32];
    uint8_t commitment_atx_id[32];
    uint8_t challenge[32];
    uint32_t num_units;
    uint64_t labels_per_unit;
} ProofMetadata;
typedef struct ScryptParams { size_t n, r, p; } ScryptParams;
typedef struct ProofConfig { uint32_t k1, k2; uint8_t pow_difficulty[32]; } ProofConfig;
typedef struct InitConfig { uint32_t min_num_units, max_num_units; uint64_t labels_per_unit; ScryptParams scrypt; } InitConfig;

typedef enum VerifyResultTag {
    VerifyOk = 0,
    VerifyInvalidIndex = 1,            /* verifying.ErrInvalidIndex{Index: invalid_index}; position in the K2 list */
    VerifyInvalidArgument = 2,
    VerifyFailedToCreateVerifier = 3,
    VerifyFailed = 4,                  /* includes an invalid k2pow */
    VerifyInvalid = 5
} VerifyResultTag;
typedef struct VerifyResult { VerifyResultTag tag; uint32_t invalid_index; } VerifyResult;

typedef struct Verifier Verifier;
/* flags: RandomX flags of the CPU library (config.PowFlags, activation/post_types.go:84-121); accepted and ignored —
 * the device always runs with the full dataset. */
VerifyResult new_verifier(uint32_t flags, Verifier **out);
void free_verifier(Verifier *verifier);
VerifyResult verify_proof(const Verifier *verifier, Proof proof, const ProofMetadata *metadata, ProofConfig cfg, InitConfig init_cfg);
VerifyResult verify_proof_index(const Verifier *verifier, Proof proof, const ProofMetadata *metadata, ProofConfig cfg,
                                InitConfig init_cfg, size_t index);
VerifyResult verify_proof_subset(const Verifier *verifier, Proof proof, const ProofMetadata *metadata, ProofConfig cfg,
                                 InitConfig init_cfg, size_t k3, const uint8_t *seed, size_t seed_len);
/* Proof over the data in `datadir` (k2pow search + proving scan, both on the device).  NULL on failure; release with
 * free_proof.  `threads` and `pow_flags` are accepted and ignored. */
Proof *generate_proof(const char *datadir, const uint8_t *challenge, ProofConfig cfg, size_t nonces, size_t threads, uint32_t pow_flags);
void free_proof(Proof *proof);

#ifdef __cplusplus
}
#endif
#endif
