/*
 * b200post.h — C ABI of the GPU-native POST label engine (libb200post.so).
 *
 * This is the drop-in boundary for go-spacemesh's POST hot path.  Every entry point is blocking,
 * thread-safe, takes plain pointers and sizes, never hands ownership of memory across the boundary and
 * returns an int status (B200POST_OK == 0).  There is NO CPU fallback inside this library: if no CUDA
 * device is usable every compute call returns B200POST_ERR_NO_DEVICE.
 *
 * What each entry point replaces in the reference (paths relative to spacemeshos/go-spacemesh):
 *
 *   b200post_providers           -> initialization.OpenCLProviders()        activation/post_supervisor.go:105-117
 *                                   (PostSetupProvider{ID, Model, DeviceType}, activation/post.go:24)
 *   b200post_labels_range        -> (*initialization.Initializer).Initialize activation/post.go:295
 *                                   = libpost `initialize(init, start, end, out, &nonce)` per ComputeBatchSize batch
 *   b200post_labels_range_multi  -> same, index range sharded over several GPUs (SURVEY.md §8e)
 *   b200post_labels_gather       -> the label recomputation inside verifying.ProofVerifier.Verify
 *                                   activation/post_verifier.go:159 (K2 / K3 / one selected index per proof)
 *   b200post_verify_vrf_nonce    -> verifying.VerifyVRFNonce                 activation/validation.go:261-282
 *   b200post_benchmark           -> initialization.Benchmark                 activation/post_supervisor.go:120-127
 *   b200post_verifier_*          -> activation.PostVerifier                  activation/interface.go:26-29,
 *                                   offloadingPostVerifier                   activation/post_verifier.go:230-390
 *
 * The libpost-compatible symbol set (new_initializer / initialize / free_initializer / ...) that
 * github.com/spacemeshos/post v0.12.9 binds through cgo is declared in post_compat.h.
 */
#ifndef B200POST_H
#define B200POST_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
    B200POST_OK = 0,
    B200POST_ERR_INVALID_ARGUMENT = 1,  /* bad pointer, N not a power of two >= 2, r/p != 1, ...           */
    B200POST_ERR_NO_DEVICE = 2,         /* no usable CUDA device / unknown provider id                       */
    B200POST_ERR_CUDA = 3,              /* a CUDA call failed; b200post_last_error() has the text            */
    B200POST_ERR_OUT_OF_MEMORY = 4,     /* not enough HBM for even one CTA per SM of ROMix scratch           */
    B200POST_ERR_CANCELLED = 5,         /* *cancel became non-zero (mirrors ctx cancel, activation/post.go:301) */
    B200POST_ERR_CLOSED = 6,            /* "verifier is closed" (activation/post_verifier.go:338,346)        */
    B200POST_ERR_INVALID_PROOF = 7,     /* verify: an index failed (verifying.ErrInvalidIndex)                */
    B200POST_ERR_EMPTY_PROOF = 8,       /* "proof indices are empty" (activation/e2e/validation_test.go:102) */
    B200POST_ERR_UNSUPPORTED = 9        /* e.g. the CPU provider id 0xffffffff: this library has no CPU path  */
};

#define B200POST_CPU_PROVIDER_ID 0xffffffffu /* systest/cluster/nodes.go:997; NOT served by this library */
#define B200POST_DEVICE_CLASS_CPU 1
#define B200POST_DEVICE_CLASS_GPU 2

typedef struct b200post_provider {
    uint32_t id;            /* CUDA device ordinal                                  */
    uint32_t device_class;  /* B200POST_DEVICE_CLASS_GPU                            */
    char model[64];         /* e.g. "NVIDIA H100 80GB HBM3"                        */
    uint64_t hbm_bytes;     /* total device memory                                  */
    uint32_t sm_count;
    uint32_t cc_major, cc_minor;
} b200post_provider;

typedef struct b200post_vrf_nonce {
    uint32_t found;         /* 1 if some label32 in the range was < difficulty (strict)            */
    uint32_t reserved;
    uint64_t index;         /* lowest index holding the minimal label32                            */
    uint8_t label32[32];    /* that label's full 32-byte scrypt output                             */
} b200post_vrf_nonce;

/* Number of usable providers; fills up to `max` entries of `out` (out may be NULL). */
int b200post_providers(b200post_provider *out, int max);

/* Thread-local text of the last error returned on this thread ("" if none). */
const char *b200post_last_error(void);

/* Engine tuning knobs (process-wide; take effect at the next call):
 *   "romix_variant"  4 pipelined (default) | 0 direct | 1 coalesced | 2 bulk(TMA) | 3 nomem (ALU probe, NOT labels)
 *   "rotate_mask"    form of the ChaCha rotates: 0 = all SHF, 1 = the 16- and 8-bit rotates as PRMT
 *   "tpb" 64|128|256|512 (64 and 512 only for the pipelined kernel; default 512) ; "dr_unroll" 4|1 ; "ctas_per_sm" 0 = as many as fit ;
 *   "max_scratch_mib" 0 = 95 % of free HBM ; "debug_skip_phase" diagnostics only.
 * Returns B200POST_ERR_INVALID_ARGUMENT for an unknown key or value. */
int b200post_set_option(const char *key, int64_t value);
int64_t b200post_get_option(const char *key);

/* label[i] = scrypt_jane(P = commitment || LE64(i) || 0^32, S = "", N = n, r = 1, p = 1, dkLen = 32)[0:16]
 * (scrypt with the ChaCha20/8 mix and HMAC-Keccak-512 PBKDF2 = libpost's label function, DESIGN.md §2) for
 * i in [start, start+count).  out16 = HOST buffer of 16*count bytes (may be NULL to discard, e.g. a
 * /dev/null init).  If vrf_difficulty != NULL (32 bytes, big-endian) the VRF-nonce scan runs over the
 * full 32-byte outputs and *nonce is filled (nonce may not be NULL then).
 * `cancel` (may be NULL) is polled between waves. */
int b200post_labels_range(uint32_t provider, const uint8_t commitment[32], uint64_t n, uint64_t start,
                          uint64_t count, uint8_t *out16, const uint8_t *vrf_difficulty,
                          b200post_vrf_nonce *nonce, const volatile int *cancel);

/* Same with the output resident in HBM: d_out16 is a DEVICE pointer on `provider` (16*count bytes,
 * 16-byte aligned) or NULL.  Nothing crosses PCIe except the optional 48-byte VRF record. */
int b200post_labels_range_dev(uint32_t provider, const uint8_t commitment[32], uint64_t n, uint64_t start,
                              uint64_t count, void *d_out16, const uint8_t *vrf_difficulty,
                              b200post_vrf_nonce *nonce, const volatile int *cancel);

/* The contiguous range split over `n_providers` devices (contiguous sub-ranges, one host thread per
 * device, VRF candidates merged on the host; no data-path collective). */
int b200post_labels_range_multi(const uint32_t *providers, int n_providers, const uint8_t commitment[32],
                                uint64_t n, uint64_t start, uint64_t count, uint8_t *out16,
                                const uint8_t *vrf_difficulty, b200post_vrf_nonce *nonce,
                                const volatile int *cancel);

/* One PROCESS per GPU (the deployment bench.py measures): each rank initialises its own contiguous shard with
 * b200post_labels_range and the ranks then agree on the VRF nonce — the path's only exchange step — with an NCCL
 * all-gather of one 64-byte record per rank and a local lexicographic arg-min (lowest label32, then lowest index).
 * Rank 0 obtains an id, hands it to the others by whatever channel the host has, every rank calls _init, then _min once
 * per batch.  libnccl.so.2 is loaded at first use; B200POST_ERR_UNSUPPORTED if it cannot be. */
typedef struct b200post_vrf_comm b200post_vrf_comm;
int b200post_vrf_comm_unique_id(uint8_t out128[128]);
int b200post_vrf_comm_init(uint32_t provider, int rank, int world, const uint8_t id128[128], b200post_vrf_comm **out);
int b200post_vrf_comm_min(b200post_vrf_comm *comm, const b200post_vrf_nonce *mine, b200post_vrf_nonce *best);
void b200post_vrf_comm_free(b200post_vrf_comm *comm);

/* labels at scattered (commitment, index) pairs: commitments = n_items x 32 bytes (HOST),
 * indices = n_items u64 (HOST), out16 = n_items x 16 bytes (HOST). */
int b200post_labels_gather(uint32_t provider, size_t n_items, const uint8_t *commitments,
                           const uint64_t *indices, uint64_t n, uint8_t *out16);

/* Same for items that share few commitments (one identity checked at K2 indices): commitments =
 * n_commitments x 32 bytes (HOST), commitment_index = n_items u32 rows into it (HOST, each < n_commitments).
 * 4 instead of 32 bytes per item cross PCIe. */
int b200post_labels_gather_indexed(uint32_t provider, size_t n_items, size_t n_commitments, const uint8_t *commitments,
                                   const uint32_t *commitment_index, const uint64_t *indices, uint64_t n,
                                   uint8_t *out16);

/* commitment = blake3(node_id || commitment_atx_id)  (hash/hash.go:16-25 primitive). */
void b200post_commitment(const uint8_t node_id[32], const uint8_t commitment_atx_id[32], uint8_t out[32]);

/* floor(2^256 / num_labels) as 32 big-endian bytes: the VRF-nonce threshold. */
void b200post_vrf_difficulty(uint64_t num_labels, uint8_t out[32]);

/* verifying.VerifyVRFNonce: recompute label32 at `nonce` and compare with the threshold for
 * num_units*labels_per_unit labels.  *valid = 1/0.
 * PARITY: the label is pinned on real data; the DECISION RULE (label32 < floor(2^256 / numLabels), strict) is a
 * recollection of spacemeshos/post and is NOT pinned — worse, the reference's own checkpoint fixture contradicts it as a
 * universal rule: 16 of its 42 recorded, network-accepted nonces are the arg-min of their POST yet lie above that
 * threshold (tests/golden/checkpoint_vrf.json, tests/test_gpu_labels.py lists them).  Do not wire this into
 * Validator.VRFNonce (activation/validation.go:261-282) before checking the rule against libpost; until then use
 * b200post_vrf_nonce_label and apply the rule the network uses. */
int b200post_verify_vrf_nonce(uint32_t provider, uint64_t nonce, const uint8_t node_id[32],
                              const uint8_t commitment_atx_id[32], uint32_t num_units,
                              uint64_t labels_per_unit, uint64_t n, int *valid);

/* The policy-free half of the above: label32 at index `nonce` of the identity's POST (through the GPU), for a caller
 * that applies its own acceptance rule. */
int b200post_vrf_nonce_label(uint32_t provider, uint64_t nonce, const uint8_t node_id[32], const uint8_t commitment_atx_id[32],
                             uint64_t n, uint8_t label32[32]);

/* ONE label32 computed on the host CPU from the same arithmetic header the kernels inline.  This is the independent
 * checker of the fault detector (the reference compares the provider's output with a CPU label and reports
 * ErrReferenceLabelMismatch, activation/post.go:299-312; b200post_setup_* does that every self_check_every batches).  It
 * is NOT a compute path: one label per call on the calling thread (~3 ms at N = 8192), nothing falls back to it. */
int b200post_reference_label(const uint8_t commitment[32], uint64_t index, uint64_t n, uint8_t out32[32]);

/* initialization.Benchmark: labels/s ("hashes/s") of a short N-scrypt run on `provider`. */
int b200post_benchmark(uint32_t provider, uint64_t n, double seconds, double *labels_per_sec);

/* Device-side instrumentation for bench.py: kernels launched by this library since load, and the
 * accumulated device time (ms, CUDA events on the launching stream) of the ROMix kernel, its launch count
 * and the label-equivalents those launches processed (a pipelined launch that fills S labels and mixes S
 * labels counts S). */
uint64_t b200post_launch_count(void);
int b200post_romix_time(uint32_t provider, double *ms_total, uint64_t *launches, double *labels, int reset);
/* Device time in ms (CUDA events recorded on the engine's own stream at the start and end of the call)
 * of the most recent labels_range* / labels_gather call on `provider`; < 0 if the provider is unusable. */
double b200post_last_call_ms(uint32_t provider);
/* Stopwatch for benchmarks: records a CUDA event on the engine's own (launching) stream; which = 0 start,
 * 1 stop.  b200post_timer_elapsed_ms waits for the stop event and returns the device time between them,
 * gaps between calls included. */
int b200post_timer_mark(uint32_t provider, int which);
double b200post_timer_elapsed_ms(uint32_t provider);
/* Labels one wave holds for scrypt-N on `provider` under the current options (= resident scratchpads). */
int b200post_wave_slots(uint32_t provider, uint64_t n, uint64_t *slots);

/* Observability: the engine's counters in the Prometheus text exposition format (the reference's metrics for this
 * path: activation/metrics/metrics.go:40-52 post_verification_waiting_total / post_verification_seconds,
 * metrics/public/public.go:19-21).  Writes at most cap-1 bytes + NUL; returns the full length needed. */
size_t b200post_metrics_text(char *buf, size_t cap);

/* Frees scratch and streams of every device (optional; also runs at library unload). */
void b200post_shutdown(void);

#ifdef __cplusplus
}
#endif
#endif /* B200POST_H */
