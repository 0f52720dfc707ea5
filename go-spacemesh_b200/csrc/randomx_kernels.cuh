// randomx_kernels.cuh — launch interface of the sm_90a RandomX kernels (k2pow).  See randomx_kernels.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "randomx_host.h"

namespace b200post {
namespace rx {

constexpr int kRcpSlots = 32;              // resolved IMUL_RCP reciprocals kept per VM and program

// Device-resident state of one batch of VMs.  The small per-VM arrays are [field][vm] (field-major: the thread-per-VM
// helper kernels touch consecutive addresses); program and reciprocals are VM-major (one warp copies them to shared memory).
struct BatchBuffers {
    uint32_t stride = 0;
    uint8_t *scratchpads = nullptr;        // stride x 2 MiB, VM-major (a VM's accesses are private and data-dependent)
    uint8_t *hot = nullptr;                // stride x 16 KiB: every VM's first 16 KiB (the "L1" level, 3 of 4 scratchpad operands),
                                           // packed into one plane that the L2 and the TLB can hold; the 2 MiB areas keep the rest
    uint2 *program = nullptr;              // [stride][256] decoded instructions (8 bytes each)
    uint64_t *rcp = nullptr;               // [stride][kRcpSlots]
    uint64_t *seed = nullptr;              // [8][stride]   the 64-byte generator state / program seed
    uint64_t *regfile = nullptr;           // [32][stride]  r0-7, f0-3, e0-3, a0-3 (lo,hi) after a program
    uint64_t *config = nullptr;            // [4][stride]   ma|mx, readReg bits|datasetOffset, eMask lo, eMask hi
    uint8_t *fprc = nullptr;               // [stride]      rounding mode carried across the 8 programs of a hash
    uint8_t *hashes = nullptr;             // stride x 32   final hashes
};

struct SuperscalarImage {                  // device copy of the 8 SuperscalarHash programs of a cache key
    const SsOp *ops = nullptr;             // concatenated
    uint32_t first[kCacheAccesses + 1] = {0};
    uint32_t address_reg[kCacheAccesses] = {0};
};

struct K2powTemplate {                     // pow[0:7] || nonce_group || challenge[0:8] || node_id  (48 bytes; post-rs layout)
    uint8_t tail[41];                      // bytes 7..47
    uint64_t start;                        // pow of VM 0
};

// dataset[item] for item in [first, first + count): spec §7.3, one thread per 64-byte item
cudaError_t launch_dataset(const uint64_t *d_cache, const SuperscalarImage &ss, uint64_t *d_dataset, uint64_t first, uint64_t count, cudaStream_t s);
// seeds: Blake2b-512 of each VM's input.  Either `inputs` (n x input_len bytes, device) or the k2pow template.
cudaError_t launch_seed_inputs(const BatchBuffers &b, uint32_t n, const uint8_t *d_inputs, uint32_t input_len, cudaStream_t s);
cudaError_t launch_seed_k2pow(const BatchBuffers &b, uint32_t n, const K2powTemplate &t, cudaStream_t s);
// AesGenerator1R: 2 MiB scratchpad per VM from its seed; the seed advances to the generator's final state
cudaError_t launch_fill_scratchpads(const BatchBuffers &b, uint32_t n, cudaStream_t s);
// AesGenerator4R -> 128 bytes of configuration + 256 instructions, decoded into the VM kernel's format
cudaError_t launch_program(const BatchBuffers &b, uint32_t n, bool first_program, cudaStream_t s);
// the VM: 2048 iterations of the 256-instruction program against scratchpad and dataset, one warp per VM.
// variant 0: 1-warp CTAs, <= 64 registers (32 VMs/SM); 1: 2-warp CTAs, <= 40 registers (48 VMs/SM, default); 2: <= 32 registers (64 VMs/SM)
cudaError_t launch_execute(const BatchBuffers &b, uint32_t n, const uint64_t *d_dataset, int variant, cudaStream_t s);
// seed = Blake2b-512(register file) for the next program of the chain
cudaError_t launch_chain_seed(const BatchBuffers &b, uint32_t n, cudaStream_t s);
// AesHash1R over the scratchpad into a0-3, then Blake2b-256(register file) -> hashes
cudaError_t launch_finalize(const BatchBuffers &b, uint32_t n, cudaStream_t s);
// k2pow: smallest VM index whose hash < difficulty (32 bytes big-endian), or 0xffffffff, into *d_found (pre-set by the caller)
cudaError_t launch_find_below(const BatchBuffers &b, uint32_t n, const uint8_t *d_difficulty, uint32_t *d_found, cudaStream_t s);
// one-time: uploads the AES tables / opcode map the kernels read
cudaError_t upload_tables();

}  // namespace rx
}  // namespace b200post
