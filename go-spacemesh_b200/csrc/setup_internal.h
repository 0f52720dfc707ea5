// setup_internal.h — what the setup sessions (setup.cu) and the stored-data VRF search (vrf_search.cu) share: the
// metadata file, the label calls of a provider choice, and the past-the-end nonce search.
#pragma once
#include <cstdint>
#include <string>

#include "../../include/b200post_setup.h"

namespace b200post {

int save_post_metadata(const std::string &dir, const b200post_post_metadata &m);

// labels [start, start + count) of scrypt-N on provider_id (a CUDA ordinal or B200POST_PROVIDER_ALL); nonce (may be
// NULL) is zeroed, then filled by the VRF scan when diff is given
int compute_labels(int64_t provider_id, uint64_t N, const uint8_t commitment[32], uint64_t start, uint64_t count, uint8_t *out,
                   const uint8_t *diff, b200post_vrf_nonce *nonce, const volatile int *cancel);

// "keep searching past numLabels until a VRF nonce is found" (SURVEY.md §8f.1): batches of `batch` labels from
// max(num_labels, md->last_position) until one is below diff; md (LastPosition, then the nonce) is saved after every
// batch, so a stopped search resumes where it stopped
int search_past_end(const std::string &dir, b200post_post_metadata *md, uint64_t num_labels, int64_t provider_id, uint64_t batch,
                    const uint8_t commitment[32], const uint8_t diff[32], const volatile int *cancel);

// b200post_search_vrf_nonce on metadata already loaded (md is updated and saved on success)
int stored_vrf_search(const std::string &dir, b200post_post_metadata *md, const b200post_vrf_search_opts &o, b200post_vrf_nonce *out,
                      const volatile int *cancel);

}  // namespace b200post
