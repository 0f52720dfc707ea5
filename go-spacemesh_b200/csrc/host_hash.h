// host_hash.h — small host-side hashing the C ABI needs outside the kernels:
// BLAKE3 for commitment = blake3(nodeID || commitmentATX) (hash/hash.go:16-25) and the VRF threshold.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>

namespace b200post {
// BLAKE3 (unkeyed) of a message of at most 1024 bytes (one chunk), `outlen` bytes of XOF output.
// Returns false if len > 1024 (multi-chunk trees are never needed on this path).
bool blake3_single_chunk(const uint8_t *msg, size_t len, uint8_t *out, size_t outlen);
void commitment_bytes(const uint8_t node_id[32], const uint8_t commitment_atx[32], uint8_t out[32]);
// floor(2^256 / num_labels), 32 big-endian bytes; saturates to 0xff..ff for num_labels <= 1.
void vrf_difficulty(uint64_t num_labels, uint8_t out[32]);
// The host order of VRF nonce candidates: the smaller big-endian label32 first, then the lower index.
inline bool vrf_less(const uint8_t a[32], uint64_t ai, const uint8_t b[32], uint64_t bi) {
    const int c = memcmp(a, b, 32);
    return c ? c < 0 : ai < bi;
}
// One label32 on the host CPU (reference_label.cpp): the fault detector's independent checker, never a compute path.
void reference_label32(const uint8_t commitment[32], uint64_t index, uint32_t n, uint8_t out[32]);
}  // namespace b200post
