// setup_internal.h — what the setup sessions (setup.cu), the stored-data VRF search (vrf_search.cu) and the merge of
// range records (range_records.cu) share: the label calls of a provider choice and the rule that settles the VRF
// nonce.  Their files are postdata_io.h's.
#pragma once
#include <cstdint>
#include <string>

#include "../../include/b200post_prove.h"

namespace b200post {

// labels [start, start + count) of scrypt-N on provider_id (a CUDA ordinal or B200POST_PROVIDER_ALL); nonce (may be
// NULL) is zeroed, then filled by the VRF scan when diff is given
int compute_labels(int64_t provider_id, uint64_t N, const uint8_t commitment[32], uint64_t start, uint64_t count, uint8_t *out,
                   const uint8_t *diff, b200post_vrf_nonce *nonce, const volatile int *cancel);

// "keep searching past numLabels until a VRF nonce is found" (SURVEY.md §8f.1): batches of `batch` labels from
// max(num_labels, md->last_position) until one is below diff; md (LastPosition, then the nonce) is saved after every
// batch, so a stopped search resumes where it stopped
int search_past_end(const std::string &dir, b200post_post_metadata *md, uint64_t num_labels, int64_t provider_id, uint64_t batch,
                    const uint8_t commitment[32], const uint8_t diff[32], const volatile int *cancel);

// The rule of an init, given the arg-min (best_index, best32) of label32 over [0, numLabels): strictly below
// floor(2^256 / numLabels) it is the nonce (LastPosition 0), else the past-the-end search on provider_id finds it
// (resumable: VrfScanPending stays set until it ends).  Clears VrfScanPending and saves md.  Pass an all-ones best32
// when no label is below the threshold.  *past_end (may be NULL): whether the search ran.
int settle_nonce(const std::string &dir, b200post_post_metadata *md, uint64_t best_index, const uint8_t best32[32], int64_t provider_id,
                 uint64_t batch, b200post_vrf_nonce *out, bool *past_end, const volatile int *cancel);

// b200post_search_vrf_nonce on metadata already loaded (md is updated and saved on success)
int stored_vrf_search(const std::string &dir, b200post_post_metadata *md, const b200post_vrf_search_opts &o, b200post_vrf_nonce *out,
                      const volatile int *cancel);

}  // namespace b200post
