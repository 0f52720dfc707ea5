/*
 * b200post_setup.h — POST data initialisation sessions on the GPU label engine (part of libb200post.so).
 *
 * Host-side mirror, behind a C ABI, of what go-spacemesh drives for POST setup:
 *   activation.PostSetupManager   PrepareInitializer / StartSession / Status / Reset   activation/post.go:245-449
 *   postSetupProvider interface                                                        activation/interface.go:114-119
 *   PostConfig / PostSetupOpts / PostSetupState                                         activation/post.go:27-61,128-137
 *   initialization.Initializer (un-vendored spacemeshos/post): postdata_N.bin files, postdata_metadata.json,
 *   resume from NumLabelsWritten, VRF nonce search incl. past the last label, LoadMetadata (post.go:373-377)
 *
 * State machine and error behaviour follow the reference's tests (activation/post_test.go:24-269):
 * StartSession without PrepareInitializer -> "post session not prepared"; a second PrepareInitializer before
 * StartSession -> "post setup session in progress"; invalid options -> error + state Error; no provider ->
 * "no provider specified" + state Error (unless the data is already complete); cancel -> state Stopped and a
 * later Prepare+Start continues where it stopped; Reset deletes the files -> NotStarted.
 *
 * The choice of the commitment ATX (database lookups, activation/post.go:373-435) stays on the Go side: it is
 * passed in, except that an existing postdata_metadata.json in data_dir wins (post.go:374-377).
 * File formats follow the published spacemeshos/post layout from memory ("parity unpinned", DESIGN.md §2).
 */
#ifndef B200POST_SETUP_H
#define B200POST_SETUP_H

#include <stddef.h>
#include <stdint.h>

#include "b200post.h"

#ifdef __cplusplus
extern "C" {
#endif

enum {                                       /* more status codes, continuing b200post.h */
    B200POST_ERR_STATE = 10,                 /* call sequence violated (text says which)                      */
    B200POST_ERR_NO_PROVIDER = 11,           /* "no provider specified" (activation/post_test.go:113)         */
    B200POST_ERR_IO = 12,                    /* file system error; b200post_last_error() has errno text       */
    B200POST_ERR_LABEL_MISMATCH = 13,        /* ErrReferenceLabelMismatch: a cross-check label differed        */
    B200POST_ERR_CONFIG_MISMATCH = 14        /* data_dir holds POST data of another identity / configuration  */
};

enum {                                       /* PostSetupState, activation/post.go:128-137 (same values) */
    B200POST_SETUP_NOT_STARTED = 1,
    B200POST_SETUP_PREPARED = 2,
    B200POST_SETUP_IN_PROGRESS = 3,
    B200POST_SETUP_STOPPED = 4,
    B200POST_SETUP_COMPLETE = 5,
    B200POST_SETUP_ERROR = 6
};

#define B200POST_PROVIDER_UNSET (-1)         /* PostSetupOpts.ProviderID == nil                                */
#define B200POST_PROVIDER_ALL (-2)           /* extension: shard every batch over all GPUs of the box         */

typedef struct b200post_post_config {        /* PostConfig, activation/post.go:27-38 */
    uint32_t min_num_units, max_num_units;
    uint64_t labels_per_unit;
    uint32_t k1, k2, k3;
    uint8_t pow_difficulty[32];
} b200post_post_config;

typedef struct b200post_setup_opts {         /* PostSetupOpts, activation/post.go:53-61 */
    const char *data_dir;
    uint32_t num_units;
    uint64_t max_file_size;                  /* bytes per postdata_N.bin; a positive multiple of 16            */
    int64_t provider_id;                     /* CUDA ordinal, B200POST_PROVIDER_UNSET or B200POST_PROVIDER_ALL */
    uint64_t scrypt_n, scrypt_r, scrypt_p;   /* config.ScryptParams; r = p = 1 required                        */
    uint64_t compute_batch_size;             /* labels per engine call; a positive multiple of 8                */
    uint32_t self_check_every;               /* cross-check one label every n batches (0 = default 16)          */
} b200post_setup_opts;

typedef struct b200post_setup_status {       /* PostSetupStatus, activation/post.go:121-125 */
    int32_t state;
    uint64_t num_labels_written;
} b200post_setup_status;

typedef struct b200post_post_metadata {      /* shared.PostMetadata as stored in postdata_metadata.json */
    uint8_t node_id[32];
    uint8_t commitment_atx_id[32];
    uint64_t labels_per_unit;
    uint32_t num_units;
    uint64_t max_file_size;
    uint64_t scrypt_n, scrypt_r, scrypt_p;
    uint32_t has_nonce;
    uint64_t nonce;                          /* VRF nonce (label index)                                         */
    uint8_t nonce_value[32];                 /* its 32-byte label                                                */
    uint64_t last_position;                  /* how far the past-the-end nonce search got                       */
} b200post_post_metadata;

typedef struct b200post_setup_manager b200post_setup_manager;

/* config.DefaultConfig()/DefaultInitOpts() equivalents used by the tests (activation/post.go:140-164). */
void b200post_default_post_config(b200post_post_config *cfg);
void b200post_default_setup_opts(b200post_setup_opts *opts);

/* NewPostSetupManager (activation/post.go:214-241). */
int b200post_setup_manager_new(const b200post_post_config *cfg, b200post_setup_manager **out);
void b200post_setup_manager_free(b200post_setup_manager *mgr);

/* PrepareInitializer: validates cfg+opts, loads or creates the metadata, finds the resume point. */
int b200post_setup_prepare_initializer(b200post_setup_manager *mgr, const b200post_setup_opts *opts,
                                       const uint8_t node_id[32], const uint8_t commitment_atx_id[32]);
/* StartSession: blocking initialisation; `cancel` (may be NULL) is the ctx.Done() analogue. */
int b200post_setup_start_session(b200post_setup_manager *mgr, const volatile int *cancel);
/* Status: callable from any thread while a session runs (NumLabelsWritten is monotone). */
int b200post_setup_get_status(b200post_setup_manager *mgr, b200post_setup_status *out);
/* Reset: deletes postdata_*.bin and the metadata of the last prepared data_dir. */
int b200post_setup_reset(b200post_setup_manager *mgr);
/* The commitment ATX the manager settled on (metadata wins over the argument of PrepareInitializer). */
int b200post_setup_commitment_atx(b200post_setup_manager *mgr, uint8_t out[32]);

/* initialization.LoadMetadata: B200POST_ERR_IO + "metadata file is missing" text if absent. */
int b200post_load_metadata(const char *data_dir, b200post_post_metadata *out);

#ifdef __cplusplus
}
#endif
#endif /* B200POST_SETUP_H */
