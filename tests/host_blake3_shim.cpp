// host_blake3_shim.cpp — a C entry point to the product's host BLAKE3 (csrc/host_hash.cpp) for the CPU tests.
#include "../go-spacemesh_b200/csrc/host_hash.h"

extern "C" int shim_blake3(const uint8_t *msg, size_t len, uint8_t *out, size_t outlen) {
    return b200post::blake3_single_chunk(msg, len, out, outlen) ? 1 : 0;
}
