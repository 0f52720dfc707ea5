// label_kernels.cuh — sm_90a kernels of the POST label path and their launch table.
//
// One label = one thread ("slot").  A *wave* is the set of slots resident on the GPU at once; every
// slot owns a private 128*N-byte ROMix scratchpad in HBM for the lifetime of the wave.
//
//   K1 pbkdf2_expand_kernel    (commitment, index) -> X[32 words]: PBKDF2-HMAC-Keccak512, scrypt step 1
//   K2 romix_kernel<VARIANT>   X <- ROMix(X) with the ChaCha20/8 BlockMix, the 99.5 % kernel (scrypt step 2)
//   K3 pbkdf2_final_kernel     X -> label32 (PBKDF2 again); 16-byte labels out via TMA bulk store; VRF candidates
//   K4 vrf_merge_kernel        per-CTA VRF candidates -> running minimum
//
// Reference anchors: activation/post.go:295 (Initialize -> labels over a contiguous range),
// activation/post_verifier.go:159 (Verify -> labels at scattered indices),
// activation/validation.go:277 (VerifyVRFNonce -> one label + VRF threshold).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "post_device.cuh"

namespace b200post {

// ROMix memory-path variants (DESIGN.md §K2):
enum RomixVariant : int {
    ROMIX_DIRECT = 0,   // each lane reads/writes its own 128-B row with 8 x 128-bit LDG/STG
    ROMIX_COALESCED = 1,// rows transposed through shared memory so that a warp moves whole 128-B lines
    ROMIX_BULK = 2,     // rows moved by the TMA unit: cp.async.bulk global<->shared + mbarrier
    ROMIX_NOMEM = 3,    // ALU ceiling probe: no scratchpad traffic (results are NOT labels)
    ROMIX_PIPELINED = 4,// two labels per thread: layer m fills while layer m-1 mixes (cp.async prefetch)
};

struct RomixParams {
    uint4 *V;            // scratch: [warp][row j][lane][8 x uint4]  (per-warp interleave)
    uint4 *X;            // state, SoA: X[k * x_stride + slot], k = 0..7
    uint32_t x_stride;   // slots in the wave buffer (multiple of 32)
    uint32_t N;          // scrypt N (power of two, >= 2)
    uint32_t n_slots;    // active slots this wave (multiple of 32)
    uint32_t flags;      // diagnostics: bit0 skip fill loop, bit1 skip mix loop (0 in production)
};

struct PipeParams {
    uint4 *V;            // scratch: [warp][parity][row j][lane][8 x uint4]  (two scratchpads per slot)
    uint4 *Xfill;        // layer being filled (initial state in, mid-state out); unused if n_fill == 0
    uint4 *Xmix;         // layer being mixed (mid-state in, final state out); unused if n_mix == 0
    uint32_t x_stride;
    uint32_t N;
    uint32_t n_fill, n_mix;   // active slots of each layer (multiples of 32)
    uint32_t fill_parity;     // which of the slot's two scratchpads the filling layer owns
    unsigned long long *cta_trace;   // diagnostics (nullptr in production): per CTA {start ns, end ns, smid}
};

struct LabelJob {
    const uint32_t *commit;     // commitments: 8 little-endian words (32 bytes) per row
    uint32_t commit_stride;     // words between the rows of consecutive slots: 0 = one shared commitment, 8 = one per slot
    const uint64_t *indices;    // nullptr => index = start + slot
    uint64_t start;
    uint32_t n_valid;           // slots that correspond to requested labels (<= n_slots)
    const uint32_t *commit_index;  // optional: per-slot row of `commit` (many items sharing few commitments); overrides commit_stride
};

struct VrfCandidate {           // 48 bytes
    uint32_t label_be[8];       // label32 as big-endian words
    uint64_t index;
    uint32_t found, pad;
};

cudaError_t launch_pbkdf2_expand(const LabelJob &job, uint4 *X, uint32_t x_stride, uint32_t n_slots, cudaStream_t s);
cudaError_t launch_romix(int variant, int rot_mask, int tpb, const RomixParams &p, cudaStream_t s);
cudaError_t launch_romix_pipe(int rot_mask, int tpb, int dr_unroll, const PipeParams &p, cudaStream_t s);
// K2s, small batches: n_slots labels spread over n_warps = romix_lowlat_warps() one-warp CTAs (p.n_slots need not be a multiple of 32)
uint32_t romix_lowlat_warps(uint32_t n_slots, int sm_count);
cudaError_t launch_romix_lowlat(int rot_mask, const RomixParams &p, uint32_t n_warps, cudaStream_t s);
// rotate-form masks compiled in (post_device.cuh ROT): 0 = all SHF, 1 = 16/8-bit rotates as PRMT
bool romix_mask_supported(int mw);
// out16: n_valid x 16 bytes (device).  vrf_difficulty_be: 8 big-endian words (device) or nullptr.
// cta_cand: one VrfCandidate per CTA (device), only touched when vrf_difficulty_be != nullptr.
cudaError_t launch_pbkdf2_final(const LabelJob &job, const uint4 *X, uint32_t x_stride, uint32_t n_slots,
                                uint8_t *out16, const uint32_t *vrf_difficulty_be, VrfCandidate *cta_cand,
                                cudaStream_t s);
cudaError_t launch_vrf_merge(const VrfCandidate *cta_cand, uint32_t n_cta, VrfCandidate *running, cudaStream_t s);
uint32_t pbkdf2_final_ctas(uint32_t n_slots);
// bytes of dynamic shared memory the ROMix variant needs per CTA
size_t romix_smem_bytes(int variant, int tpb);
// occupancy query helper: max resident CTAs/SM for (variant, mask, tpb)
int romix_max_ctas_per_sm(int variant, int rot_mask, int tpb, int dr_unroll);
const char *romix_variant_name(int variant);

}  // namespace b200post
