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
    uint32_t vrf_scan_pending;               /* "VrfScanPending": some stored labels were written by a file-range
                                                session and never VRF-scanned; the nonce must come from the stored
                                                data (b200post_search_vrf_nonce, or a full session's final step)   */
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
/*
 * PrepareInitializer restricted to postdata files [from_file, to_file]; to_file = -1 means the POST's last file
 * (postcli -fromFile / -toFile: one POST initialised on several machines).  prepare_initializer is (0, -1).
 * from_file <= to_file < n_files = ceil(NumUnits * LabelsPerUnit / (MaxFileSize / 16)), else INVALID_ARGUMENT.
 * A range short of the whole POST covers labels [from * perFile, min((to + 1) * perFile, numLabels)); it resumes from
 * from_file (full files, then one partial file) and never opens, creates or writes a file outside the range; the
 * status counts the range's labels.  It records no VRF nonce and runs no past-the-end search (a range's arg-min is not
 * the POST's).  If the metadata has no nonce yet, prepare sets "VrfScanPending": copy the files of every range into
 * one directory with any one metadata file, then b200post_search_vrf_nonce (or a full session) finds the nonce.  If
 * the metadata already has a nonce (re-initialising a damaged or lost file), it is kept and no marker is set.
 */
int b200post_setup_prepare_files(b200post_setup_manager *mgr, const b200post_setup_opts *opts, const uint8_t node_id[32],
                                 const uint8_t commitment_atx_id[32], uint64_t from_file, int64_t to_file);
/* StartSession: blocking initialisation; `cancel` (may be NULL) is the ctx.Done() analogue.  A full session on data
 * whose metadata has VrfScanPending runs b200post_search_vrf_nonce's stored-data search once every label is on disk. */
int b200post_setup_start_session(b200post_setup_manager *mgr, const volatile int *cancel);
/* Status: callable from any thread while a session runs (NumLabelsWritten is monotone). */
int b200post_setup_get_status(b200post_setup_manager *mgr, b200post_setup_status *out);
/* Reset: deletes postdata_*.bin and the metadata of the last prepared data_dir. */
int b200post_setup_reset(b200post_setup_manager *mgr);
/* The commitment ATX the manager settled on (metadata wins over the argument of PrepareInitializer). */
int b200post_setup_commitment_atx(b200post_setup_manager *mgr, uint8_t out[32]);

/* initialization.LoadMetadata: B200POST_ERR_IO + "metadata file is missing" text if absent. */
int b200post_load_metadata(const char *data_dir, b200post_post_metadata *out);

/*
 * Checking stored POST data (postcli -verify; spacemeshos/post verifying.VerifyPos, from memory, unpinned):
 * recompute a share of each file's labels on the GPU and compare them with the bytes in postdata_N.bin.
 * Inputs come from postdata_metadata.json (commitment = blake3(NodeId || CommitmentAtxId), N, file size, label count).
 * Host-side errors come first: bad arguments -> INVALID_ARGUMENT; no metadata -> ERR_IO "metadata file is missing";
 * a file whose size differs from what the metadata implies (the last file may be short) -> ERR_IO "incomplete";
 * then, without a GPU, ERR_NO_DEVICE (there is no CPU path).  Any mismatch, or a VRF nonce whose recomputed label
 * differs from NonceValue, returns B200POST_ERR_LABEL_MISMATCH with `out` filled.  When every checked label matches but the metadata has no VRF nonce
 * (initialisation stopped before finding it), the call returns B200POST_ERR_STATE with `out` filled, nonce_ok = 0 and
 * argmin_checked = 0.  A set *cancel returns B200POST_ERR_CANCELLED with partial counts.
 * A file of L labels contributes max(1, floor(L * fraction / 100)) distinct positions (all of them at 100), a
 * deterministic function of (seed, file index), so shards and re-runs check the same labels.
 */
typedef struct b200post_verify_pos_opts {
    int64_t provider_id;         /* CUDA ordinal or B200POST_PROVIDER_ALL                                  */
    double fraction;             /* percent of each file's labels, (0, 100]; 100 = every label             */
    uint64_t from_file;          /* first postdata_N.bin                                                    */
    int64_t to_file;             /* last file, inclusive; -1 = the POST's last file                         */
    uint64_t seed;               /* sample seed; 0 = draw one from the OS (returned in the result)          */
    volatile uint64_t *progress; /* optional: labels checked so far                                         */
} b200post_verify_pos_opts;

typedef struct b200post_verify_pos_result {
    uint64_t files_checked, labels_checked, mismatches, seed;
    uint32_t nonce_ok;                    /* label32 at metadata Nonce == NonceValue (0 when there is no nonce)       */
    uint32_t argmin_checked, argmin_ok;   /* full check of every file with a nonce: the fused VRF scan agrees with it  */
    uint32_t n_reported;
    uint64_t bad_index[64];               /* lowest mismatching global label indices, ascending                      */
} b200post_verify_pos_result;

/* provider 0, fraction 0.2, all files, seed 0 */
void b200post_default_verify_pos_opts(b200post_verify_pos_opts *o);
int b200post_verify_pos(const char *data_dir, const b200post_verify_pos_opts *o, b200post_verify_pos_result *out,
                        const volatile int *cancel);
/* Which positions (within the file, ascending) a seed checks, for reproducing a run: *n = the sample size; out
 * (may be NULL to ask for the size only) receives them when cap >= *n, else INVALID_ARGUMENT. */
int b200post_verify_pos_sample(uint64_t seed, uint64_t file, uint64_t labels_in_file, double fraction,
                               uint64_t *out, uint64_t cap, uint64_t *n);

/*
 * The VRF nonce from stored labels (postcli -searchForNonce, recalled, unpinned): for a POST whose files were written
 * by several file-range sessions, none of which saw every label.  The rule is the one an init applies: the nonce is
 * the lowest label32 (big-endian), lowest index on ties, recorded only if strictly below floor(2^256 / numLabels);
 * otherwise the past-the-end search runs from numLabels in compute_batch_size batches.
 * The arg-min of label32 is decided by its first 16 bytes, which are what is stored: the files are streamed through
 * the GPU (K8) at 16 B per label, and only the labels at the lowest stored prefix have their label32 recomputed.
 * One of those whose recomputed first 16 bytes differ from the stored ones means damaged data: LABEL_MISMATCH with
 * the index in the error text, metadata untouched.  A label damaged upwards is invisible to a scan that trusts the
 * stored bytes: `b200postcli -verify -fraction 100` (b200post_verify_pos) is the check for that.
 * Host errors first: no metadata -> ERR_IO; a missing or short file -> ERR_IO "incomplete"; then ERR_NO_DEVICE
 * without a GPU (no CPU path).  On success Nonce / NonceValue / LastPosition are written as a single uninterrupted
 * init would have written them, and VrfScanPending is cleared.
 */
typedef struct b200post_vrf_search_opts {
    int64_t provider_id;           /* CUDA ordinal or B200POST_PROVIDER_ALL (scan on the first device, past-the-end search on all) */
    uint64_t compute_batch_size;   /* batch of the past-the-end search; 0 = 2^20. The same batch as a single init gives the same nonce */
    uint64_t chunk_labels;         /* labels per H2D chunk; 0 = 2^22 (64 MiB), as the prover; at most 2^26 */
    volatile uint64_t *progress;   /* optional: labels scanned */
} b200post_vrf_search_opts;
/* provider 0, batch 2^20, chunk 2^22, no progress */
void b200post_default_vrf_search_opts(b200post_vrf_search_opts *o);
int b200post_search_vrf_nonce(const char *data_dir, const b200post_vrf_search_opts *o, b200post_vrf_nonce *out,
                              const volatile int *cancel);

/*
 * Block checksums (DESIGN.md §3g).  A block is B = 2^16 labels (1 MiB) of one postdata_N.bin, aligned to the file's
 * first label; the file's last block may be shorter.  Its digest is unkeyed BLAKE3 of its bytes (32 bytes).  The
 * sidecar postdata_N.sum holds the digests of the file's labels [0, covered): whole blocks, except possibly the last,
 * which covers [floor((covered - 1) / B) * B, covered).  Sidecars are made only from labels computed on a device, never
 * from bytes read back (b200post_write_sums: only after every label of the file was recomputed and matched), so no
 * session makes one wrong; labels past `covered` are unchecked.  libpost's readers look only at postdata_<N>.bin
 * (recalled, unpinned), so the sidecars do not disturb them.
 */

/* The digests of `count` labels (count x 16 bytes, host memory) split into blocks of 2^16 labels from the first, the
 * last one short: ceil(count / 2^16) x 32 bytes into digests32, hashed on CUDA ordinal `provider`. */
int b200post_label_block_digests(uint32_t provider, const uint8_t *labels16, uint64_t count, uint8_t *digests32);

/* Ask the prepared session (whole POST or file range, with or without an initial proof or a range record) to write
 * postdata_N.sum for every file it writes, from the labels it computes, hashed on its first device after the
 * self-check.  A sidecar is saved after every batch that completes a block, at the end of each file, and when the
 * session stops or fails.  On resume, the whole blocks of a usable sidecar below the labels on disk are kept and the
 * rest of those labels (from label 0 when the sidecar is absent, damaged or made for another identity, N, file size or
 * file) is recomputed and hashed first, not read back; the initial-proof scan, the VRF scan and a range record never
 * see them.  The labels, the metadata, initial_post.json and range records are byte-identical to a session without
 * the request.  Call between prepare and start; prepare clears the request. */
int b200post_setup_request_checksums(b200post_setup_manager *mgr);

typedef struct b200post_sums_opts {
    int64_t provider_id;         /* check: a CUDA ordinal; write: a CUDA ordinal or B200POST_PROVIDER_ALL      */
    uint64_t from_file;          /* first postdata_N.bin                                                      */
    int64_t to_file;             /* last file, inclusive; -1 = the POST's last file                           */
    volatile uint64_t *progress; /* optional: labels hashed (check) or recomputed and compared (write) so far */
    uint32_t repair;             /* check only: 1 = rewrite each bad block from its recomputation             */
} b200post_sums_opts;

typedef struct b200post_sums_block {
    uint64_t first_label;        /* global label index of the block's first label */
    uint64_t count;              /* its labels                                     */
} b200post_sums_block;

typedef struct b200post_sums_result {
    uint64_t files_checked;      /* check: files with a usable sidecar; write: files given one                */
    uint64_t files_unchecked;    /* check: files without a usable sidecar; write: files with a mismatch       */
    uint64_t labels_checked, labels_unchecked;
    uint64_t bytes_read;
    uint64_t blocks_checked, bad_blocks, repaired_blocks;
    uint32_t n_reported;
    uint32_t reserved;
    b200post_sums_block bad[64]; /* the lowest bad blocks, ascending                                          */
} b200post_sums_result;

/* provider 0, all files, no progress, no repair */
void b200post_default_sums_opts(b200post_sums_opts *o);

/*
 * Check stored labels against their sidecars at storage speed: the covered labels of files [from_file, to_file] are
 * read (pinned, double-buffered), hashed on the device and compared block by block.  Host checks first, in order:
 * bad arguments -> INVALID_ARGUMENT; no metadata -> ERR_IO; a missing or short file -> ERR_IO "incomplete"; a file
 * without a usable sidecar is counted unchecked, and when no label of the range is covered -> ERR_STATE "no checksums";
 * then UNSUPPORTED for the CPU id or NO_DEVICE.  Returns LABEL_MISMATCH when a block differs (the lowest 64 reported),
 * else ERR_STATE when labels were unchecked, else OK; `out` is filled in each case.
 * repair = 1: each bad block is recomputed under the metadata's N and hashed; its digest must equal the sidecar's (else
 * LABEL_MISMATCH "recomputed block disagrees with its checksum", nothing written), then it is written with pwrite,
 * fdatasync'ed, read back and hashed again.  Repaired blocks no longer count towards LABEL_MISMATCH.  Repair never
 * touches the metadata, the nonce, initial_post.json or records; a missing or short file is a range session's job.
 */
int b200post_check_sums(const char *data_dir, const b200post_sums_opts *o, b200post_sums_result *out, const volatile int *cancel);

/*
 * Sidecars for data that has none (written by libpost, earlier sessions, or without the request): the full check of
 * b200post_verify_pos (fraction 100, every label recomputed and compared) over files [from_file, to_file], and for each
 * file whose labels all match, the sidecar from the digests of those verified bytes, byte-identical to the one an init
 * with checksums writes.  A file with a mismatch gets none and is counted in files_unchecked, its damaged blocks
 * reported (from the lowest mismatching labels of each compare call): LABEL_MISMATCH.  Host checks as above (no
 * sidecar needed).  Costs one full check.
 */
int b200post_write_sums(const char *data_dir, const b200post_sums_opts *o, b200post_sums_result *out, const volatile int *cancel);

#ifdef __cplusplus
}
#endif
#endif /* B200POST_SETUP_H */
