// vrf_verify.cu — K9, the device verdict of batched VRF-nonce checks (b200post_verify_vrf_nonces and the verifier's
// VRF jobs, verifier.cu).
//
// verifying.VerifyVRFNonce (activation/validation.go:261-282) recomputes ONE label per check: the label at the nonce.
// The verifier recomputes the labels of every check in a batch with the same gather as its proofs, through K3w, so both
// 16-byte halves of each label32 are in HBM.  K9 then judges each check against its own threshold
// floor(2^256 / numLabels) (items differ in num_units x labels_per_unit) with the VRF order of post_device.cuh, and
// writes the verdict and the compact label32 for one D2H copy.  The rule (label32 < threshold, strict) is the UNPINNED
// one of b200post_verify_vrf_nonce; label32 goes back with it so that a caller can apply the network's own rule.
#include "label_kernels.cuh"

namespace b200post {

// one thread per check; lo16/hi16 are the gather's outputs, the checks' labels start at position `first`
__global__ void __launch_bounds__(256) vrf_judge_kernel(const uint4 *__restrict__ lo16, const uint4 *__restrict__ hi16, uint32_t first,
                                                        uint32_t n_items, const uint4 *__restrict__ threshold_be,
                                                        uint8_t *__restrict__ valid, uint4 *__restrict__ label32_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_items) return;
    const uint4 lo = lo16[first + i], hi = hi16[first + i];
    const uint4 t0 = threshold_be[2 * (size_t)i], t1 = threshold_be[2 * (size_t)i + 1];
    // the stored halves are the big-endian serialisation of the label words (K3w): back to words for the compare
    const uint32_t lab[8] = {bswap32(lo.x), bswap32(lo.y), bswap32(lo.z), bswap32(lo.w),
                             bswap32(hi.x), bswap32(hi.y), bswap32(hi.z), bswap32(hi.w)};
    const uint32_t thr[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
    valid[i] = cand_less(lab, 0, thr, 0) ? 1 : 0;   // equal indices: strict '<' on the label
    label32_out[2 * (size_t)i] = lo;
    label32_out[2 * (size_t)i + 1] = hi;
}

cudaError_t launch_vrf_judge(const uint4 *lo16, const uint4 *hi16, uint32_t first, uint32_t n_items, const uint4 *threshold_be,
                             uint8_t *valid, uint4 *label32_out, cudaStream_t s) {
    if (n_items == 0) return cudaSuccess;
    vrf_judge_kernel<<<(n_items + 255) / 256, 256, 0, s>>>(lo16, hi16, first, n_items, threshold_be, valid, label32_out);
    return cudaGetLastError();
}

}  // namespace b200post
