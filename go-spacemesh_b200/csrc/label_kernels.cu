// label_kernels.cu — hand-written sm_90a kernels for the POST label path (see label_kernels.cuh).
#include "label_kernels.cuh"

namespace b200post {

// =================================================================================================
// PTX helpers
// =================================================================================================
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Scratchpad accesses are streaming (.cs = evict-first): V is written once and read about once, and a
// wave's scratch (tens of GiB) never fits the 50 MB L2.  (Default and .cg policies measured the same.)
__device__ __forceinline__ uint4 ld_stream(const uint4 *p) {
    uint4 v;
    asm volatile("ld.global.cs.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_stream(uint4 *p, const uint4 &v) {
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// Ampere-style async copy global -> shared, 16 B per lane, L2 only (SASS: LDGSTS)
__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_smem), "l"(src) : "memory");
}
// Same with the 64-bit source address given as {lo, hi} + immediate: scratchpad regions never cross a 4 GiB
// boundary (the engine aligns V to the region size), so per-row address math is one 32-bit IMAD on the
// fmaheavy pipe instead of 64-bit IADD3/IMAD.WIDE chains on the saturated alu pipe.
template <int IMM>
__device__ __forceinline__ void cp_async16_lohi(uint32_t dst_smem, uint32_t lo, uint32_t hi) {
    asm volatile("{\n\t.reg .b64 a;\n\tmov.b64 a, {%1, %2};\n\tcp.async.cg.shared.global [%0], [a+%3], 16;\n\t}"
                 ::"r"(dst_smem), "r"(lo), "r"(hi), "n"(IMM) : "memory");
}
template <int IMM>
__device__ __forceinline__ void st_stream_lohi(uint32_t lo, uint32_t hi, const uint4 &v) {
    asm volatile("{\n\t.reg .b64 a;\n\tmov.b64 a, {%0, %1};\n\tst.global.cs.v4.u32 [a+%2], {%3,%4,%5,%6};\n\t}"
                 ::"r"(lo), "r"(hi), "n"(IMM), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint32_t mad_u32(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void sts128(uint32_t a, const uint4 &v) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
// TMA 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// TMA 1-D bulk copy shared -> global, tracked by the thread's bulk async-group
__device__ __forceinline__ void bulk_s2g(void *dst, uint32_t src_smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src_smem), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N_PENDING>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N_PENDING) : "memory"); }
template <int N_PENDING>
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N_PENDING) : "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// chunk k (0..7) of a 32-word row held as lo[16] || hi[16]
#define ROW_CHUNK(lo, hi, k) \
    ((k) < 4 ? make_uint4(lo[4 * (k)], lo[4 * (k) + 1], lo[4 * (k) + 2], lo[4 * (k) + 3]) \
             : make_uint4(hi[4 * (k) - 16], hi[4 * (k) - 15], hi[4 * (k) - 14], hi[4 * (k) - 13]))
__device__ __forceinline__ void set_chunk(uint32_t (&lo)[16], uint32_t (&hi)[16], int k, const uint4 &v) {
    // k is always a compile-time constant after unrolling
    if (k < 4) { lo[4 * k] = v.x; lo[4 * k + 1] = v.y; lo[4 * k + 2] = v.z; lo[4 * k + 3] = v.w; }
    else { hi[4 * k - 16] = v.x; hi[4 * k - 15] = v.y; hi[4 * k - 14] = v.z; hi[4 * k - 13] = v.w; }
}

// the commitment of `slot` as 8 little-endian words
__device__ __forceinline__ void load_commit(const LabelJob &job, uint32_t slot, uint32_t (&c)[8]) {
    const uint32_t *p = job.commit_index ? job.commit + 8 * (size_t)job.commit_index[slot] : job.commit + (size_t)job.commit_stride * slot;
#pragma unroll
    for (int k = 0; k < 8; k++) c[k] = p[k];
}
__device__ __forceinline__ uint64_t slot_index(const LabelJob &job, uint32_t slot) {
    if (job.indices) return slot < job.n_valid ? job.indices[slot] : 0;
    return job.start + slot;
}

// =================================================================================================
// K1: PBKDF2 expand  (8 Keccak-f[1600] permutations per label)
// =================================================================================================
__global__ void __launch_bounds__(128) pbkdf2_expand_kernel(LabelJob job, uint4 *__restrict__ X, uint32_t x_stride, uint32_t n_slots) {
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= n_slots) return;
    uint32_t c[8];
    load_commit(job, slot < job.n_valid ? slot : 0, c);
    uint32_t lo[16], hi[16];
    label_expand(c, slot_index(job, slot), lo, hi);
#pragma unroll
    for (int k = 0; k < 8; k++) X[(size_t)k * x_stride + slot] = ROW_CHUNK(lo, hi, k);
}

// =================================================================================================
// K2: ROMix.  V layout (all variants): per-warp interleave, row j of lane t at
//     V + ((warp * N + j) * 32 + t) * 8 uint4      => in phase 1 a warp writes 4 KiB contiguous per j,
//     and one lane's phase-2 reads stay inside its warp's 128*N*32-byte region (TLB-friendly).
// COALESCED and BULK store rows "swizzled": chunk k of lane t sits at chunk position k ^ (t & 7).  V is
// private scratch, so any layout is legal as long as reads undo it; the swizzle makes the dense
// 32 x 128-B shared-memory tile bank-conflict-free in both the row-wise and the transposed access.
// =================================================================================================
template <int VARIANT, int MW, int TPB>
__global__ void __launch_bounds__(TPB) romix_kernel(const RomixParams p) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const uint32_t slot = blockIdx.x * TPB + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31, warp_in_cta = threadIdx.x >> 5;
    if (slot >= p.n_slots) return;   // n_slots is a multiple of 32: whole warps leave together
    const uint32_t N = p.N, mask = N - 1;
    // diagnostics only (b200post_set_option("debug_skip_phase")): bit0 skips the fill loop, bit1 the mix loop
    const uint32_t n1 = (p.flags & 1) ? 0 : N, n2 = (p.flags & 2) ? 0 : N;

    uint32_t lo[16], hi[16];
#pragma unroll
    for (int k = 0; k < 8; k++) set_chunk(lo, hi, k, p.X[(size_t)k * p.x_stride + slot]);

    uint4 *const Vw = p.V + (size_t)(slot >> 5) * N * 256;   // this warp's region; row j at Vw + j*256
    const uint32_t swz = lane & 7;

    if (VARIANT == ROMIX_DIRECT) {
        uint4 *const Vt = Vw + lane * 8;
        for (uint32_t i = 0; i < n1; i++) {
#pragma unroll
            for (int k = 0; k < 8; k++) st_stream(Vt + (size_t)i * 256 + k, ROW_CHUNK(lo, hi, k));
            blockmix_r1<MW>(lo, hi);
        }
        for (uint32_t i = 0; i < n2; i++) {
            const uint32_t j = hi[0] & mask;
            uint32_t vlo[16], vhi[16];
#pragma unroll
            for (int k = 0; k < 8; k++) set_chunk(vlo, vhi, k, ld_stream(Vt + (size_t)j * 256 + k));
            blockmix_r1_xor<MW>(lo, hi, vlo, vhi);
        }
    } else if (VARIANT == ROMIX_COALESCED) {
        const uint32_t tile = smem_u32(smem_raw) + warp_in_cta * 4096;
        const uint32_t own = tile + lane * 128;
        const uint32_t tr_row = lane >> 3, tr_c = lane & 7;   // transposed role: row k*4+tr_row, chunk position tr_c
        for (uint32_t i = 0; i < n1; i++) {
#pragma unroll
            for (int k = 0; k < 8; k++) sts128(own + ((k ^ swz) << 4), ROW_CHUNK(lo, hi, k));
            __syncwarp();
            uint4 *const dst = Vw + (size_t)i * 256 + lane;   // + k*32: the warp writes 512 contiguous bytes per k
#pragma unroll
            for (int k = 0; k < 8; k++) st_stream(dst + k * 32, lds128(tile + (k * 4 + tr_row) * 128 + (tr_c << 4)));
            __syncwarp();
            blockmix_r1<MW>(lo, hi);
        }
        for (uint32_t i = 0; i < n2; i++) {
            const uint32_t j = hi[0] & mask;
            uint4 t[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const uint32_t jr = __shfl_sync(0xffffffffu, j, k * 4 + tr_row);
                t[k] = ld_stream(Vw + (size_t)jr * 256 + k * 32 + lane);
            }
#pragma unroll
            for (int k = 0; k < 8; k++) sts128(tile + (k * 4 + tr_row) * 128 + (tr_c << 4), t[k]);
            __syncwarp();
            uint32_t vlo[16], vhi[16];
#pragma unroll
            for (int k = 0; k < 8; k++) set_chunk(vlo, vhi, k, lds128(own + ((k ^ swz) << 4)));
            __syncwarp();
            blockmix_r1_xor<MW>(lo, hi, vlo, vhi);
        }
    } else if (VARIANT == ROMIX_BULK) {
        // per warp: two 4-KiB tiles (double-buffered bulk stores in phase 1) + one mbarrier
        constexpr uint32_t WARPS = TPB / 32;
        const uint32_t tile0 = smem_u32(smem_raw) + warp_in_cta * 8192;
        const uint32_t bar = smem_u32(smem_raw) + WARPS * 8192 + warp_in_cta * 8;
        if (lane == 0) mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        __syncwarp();
        for (uint32_t i = 0; i < n1; i++) {
            const uint32_t tile = tile0 + (i & 1) * 4096;
            if (lane == 0) bulk_wait_read<1>();   // the store issued two iterations ago has drained this tile
            __syncwarp();
#pragma unroll
            for (int k = 0; k < 8; k++) sts128(tile + lane * 128 + ((k ^ swz) << 4), ROW_CHUNK(lo, hi, k));
            fence_proxy_async_smem();
            __syncwarp();
            if (lane == 0) { bulk_s2g(Vw + (size_t)i * 256, tile, 4096); bulk_commit(); }
            blockmix_r1<MW>(lo, hi);
        }
        if (lane == 0) bulk_wait_all<0>();
        __syncwarp();
        const uint32_t own = tile0 + lane * 128;
        uint32_t parity = 0;
        for (uint32_t i = 0; i < n2; i++) {
            const uint32_t j = hi[0] & mask;
            if (lane == 0) mbar_expect_tx(bar, 4096);
            __syncwarp();
            bulk_g2s(own, Vw + (size_t)j * 256 + lane * 8, 128, bar);
            mbar_wait(bar, parity);
            parity ^= 1;
            uint32_t vlo[16], vhi[16];
#pragma unroll
            for (int k = 0; k < 8; k++) set_chunk(vlo, vhi, k, lds128(own + ((k ^ swz) << 4)));
            blockmix_r1_xor<MW>(lo, hi, vlo, vhi);
        }
    } else {   // ROMIX_NOMEM: same arithmetic, no scratchpad (ALU ceiling probe only)
        for (uint32_t i = 0; i < n1; i++) blockmix_r1<MW>(lo, hi);
        for (uint32_t i = 0; i < n2; i++) {
            uint32_t vlo[16], vhi[16];
#pragma unroll
            for (int k = 0; k < 16; k++) { vlo[k] = hi[(k + 1) & 15] + i; vhi[k] = lo[(k + 3) & 15]; }
            blockmix_r1_xor<MW>(lo, hi, vlo, vhi);
        }
    }
#pragma unroll
    for (int k = 0; k < 8; k++) p.X[(size_t)k * p.x_stride + slot] = ROW_CHUNK(lo, hi, k);
}

// =================================================================================================
// K2s: low-latency ROMix for SMALL batches (one proof = K2 = 37 labels; a VRF-nonce check = 1 label).
// A label is a serial chain — 2N BlockMix steps of two dependent ChaCha20/8 cores, ~100 dependent integer operations
// each — so its latency floor on this clock is ~7 ms however many lanes are thrown at it (splitting a core over four
// lanes leaves the chain as long and adds shuffles: a single lane already issues the four independent quarter rounds
// back to back).  What CAN be removed is everything the throughput kernel adds for a full wave: here a label gets a
// lane, labels are spread over as many WARPS as there are scheduler slots (SMs x 4) so that every label's warp issues
// every cycle, and for a proof's K2 = 37 labels the scratchpad rows (n MiB in total) stay in the 50 MB L2, so the
// dependent phase-2 read is an L2 hit.  Slot s is handled by lane s / W of warp s % W (W = warps launched); V is private scratch, label-major here:
// row j of slot s at V + (s * N + j) * 8 uint4 (n x 128*N bytes in total, whatever W is).
// =================================================================================================
__device__ __forceinline__ uint4 ld_l2(const uint4 *p) {
    uint4 v;
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_l2(uint4 *p, const uint4 &v) {
    asm volatile("st.global.cg.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
template <int MW>
__global__ void __launch_bounds__(32) romix_lowlat_kernel(const RomixParams p, uint32_t n_warps) {
    const uint32_t lane = threadIdx.x, warp = blockIdx.x;
    const uint32_t slot = lane * n_warps + warp;
    if (slot >= p.n_slots) return;
    const uint32_t N = p.N, mask = N - 1;
    uint32_t lo[16], hi[16];
#pragma unroll
    for (int k = 0; k < 8; k++) set_chunk(lo, hi, k, p.X[(size_t)k * p.x_stride + slot]);
    uint4 *const Vt = p.V + (size_t)slot * N * 8;          // label-major: 128*N contiguous bytes per label
    for (uint32_t i = 0; i < N; i++) {
#pragma unroll
        for (int k = 0; k < 8; k++) st_l2(Vt + (size_t)i * 8 + k, ROW_CHUNK(lo, hi, k));
        blockmix_r1<MW>(lo, hi);
    }
    for (uint32_t i = 0; i < N; i++) {
        const uint32_t j = hi[0] & mask;
        uint32_t vlo[16], vhi[16];
#pragma unroll
        for (int k = 0; k < 8; k++) set_chunk(vlo, vhi, k, ld_l2(Vt + (size_t)j * 8 + k));
        blockmix_r1_xor<MW>(lo, hi, vlo, vhi);
    }
#pragma unroll
    for (int k = 0; k < 8; k++) p.X[(size_t)k * p.x_stride + slot] = ROW_CHUNK(lo, hi, k);
}

// =================================================================================================
// K2p: pipelined ROMix.  Every thread advances TWO labels per step: the label of layer m is in its fill
// loop (V[i] <- X; X <- BlockMix(X)) while the label of layer m-1 is in its mix loop
// (X <- BlockMix(X ^ V[Integerify(X)])).  The mix loop's dependent HBM read (~0.6-1.5 us) is issued
// with cp.async at the top of the step and lands in shared memory while the fill label's BlockMix
// keeps the integer pipes busy.
// Each slot owns two scratchpads (parity = layer & 1).  The mid-state of a filled label travels to the
// next launch through the layer's X buffer, so consecutive launches form one software pipeline:
//     launch m:  K1(layer m) -> K2p{mix layer m-1, fill layer m} -> K3(layer m-1)
// =================================================================================================
template <int MW, int TPB, int DR_UNROLL>
__global__ void __launch_bounds__(TPB) romix_pipe_kernel(const PipeParams p) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const uint32_t slot = blockIdx.x * TPB + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31, warp_in_cta = threadIdx.x >> 5;
    const bool do_fill = slot < p.n_fill, do_mix = slot < p.n_mix;   // multiples of 32: warp-uniform
    if (!do_fill && !do_mix) return;
    if (p.cta_trace && threadIdx.x == 0) {
        unsigned long long t; uint32_t sm;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
        p.cta_trace[3 * (size_t)blockIdx.x] = t; p.cta_trace[3 * (size_t)blockIdx.x + 2] = sm;
    }
    const uint32_t N = p.N, mask = N - 1;
    const uint32_t tile_f = smem_u32(smem_raw) + warp_in_cta * 8192, tile_m = tile_f + 4096;
    const uint32_t own_f = tile_f + lane * 128, own_m = tile_m + lane * 128;
    const uint32_t swz = lane & 7, tr_row = lane >> 3, tr_c = lane & 7;
    const size_t warp = slot >> 5;
    // this lane's base addresses inside the two scratchpad regions of its warp, as {lo, hi}: a region is
    // N * 4 KiB, V is aligned to the region size and N <= 2^20, so `hi` is constant within a region
    const uint64_t vf64 = (uint64_t)(p.V + (warp * 2 + p.fill_parity) * (size_t)N * 256 + lane);         // written
    const uint64_t vm64 = (uint64_t)(p.V + (warp * 2 + (p.fill_parity ^ 1)) * (size_t)N * 256 + lane);   // read
    const uint32_t vf_hi = (uint32_t)(vf64 >> 32), vm_lo = (uint32_t)vm64, vm_hi = (uint32_t)(vm64 >> 32);
    uint32_t vf_cur = (uint32_t)vf64;   // low word of row i's address for this lane; +4096 per step

    uint32_t lo_f[16], hi_f[16], lo_m[16], hi_m[16];
    if (do_fill) {
#pragma unroll
        for (int k = 0; k < 8; k++) set_chunk(lo_f, hi_f, k, p.Xfill[(size_t)k * p.x_stride + slot]);
    }
    if (do_mix) {
#pragma unroll
        for (int k = 0; k < 8; k++) set_chunk(lo_m, hi_m, k, p.Xmix[(size_t)k * p.x_stride + slot]);
    }
    // lane whose j this lane needs for its k-th transposed copy (loop-invariant)
    uint32_t src_lane[8];
#pragma unroll
    for (int k = 0; k < 8; k++) src_lane[k] = k * 4 + tr_row;
    const uint32_t tile_m_tr = tile_m + tr_row * 128 + (tr_c << 4);
    const uint32_t tile_f_tr = tile_f + tr_row * 128 + (tr_c << 4);

    // issue the mix label's row read: 8 x (4 rows x 128 B) per warp, straight into the shared tile
#define MIX_PREFETCH_K(k) \
    cp_async16_lohi<(k) * 512>(tile_m_tr + (k) * 512, mad_u32(__shfl_sync(0xffffffffu, j, src_lane[k]), 4096u, vm_lo), vm_hi);
    auto mix_prefetch = [&]() {
        const uint32_t j = hi_m[0] & mask;
        MIX_PREFETCH_K(0) MIX_PREFETCH_K(1) MIX_PREFETCH_K(2) MIX_PREFETCH_K(3)
        MIX_PREFETCH_K(4) MIX_PREFETCH_K(5) MIX_PREFETCH_K(6) MIX_PREFETCH_K(7)
        cp_async_commit();
    };
    // write the fill label's row i: own row -> tile (swizzled), tile -> HBM as 8 x 512 contiguous bytes
#define FILL_STORE_K(k) st_stream_lohi<(k) * 512>(vf_cur, vf_hi, lds128(tile_f_tr + (k) * 512));
    auto fill_store = [&]() {
#pragma unroll
        for (int k = 0; k < 8; k++) sts128(own_f + ((k ^ swz) << 4), ROW_CHUNK(lo_f, hi_f, k));
        __syncwarp();
        FILL_STORE_K(0) FILL_STORE_K(1) FILL_STORE_K(2) FILL_STORE_K(3)
        FILL_STORE_K(4) FILL_STORE_K(5) FILL_STORE_K(6) FILL_STORE_K(7)
        __syncwarp();
        vf_cur = mad_u32(1u, 4096u, vf_cur);
    };

    // One loop serves all three launch shapes (fill+mix in steady state, fill only for the first layer,
    // mix only for the drain).  The mix label's row for step i is requested at the end of step i-1 and
    // lands in shared memory while this step's fill BlockMix occupies the integer pipes.
    if (do_mix) mix_prefetch();
    for (uint32_t i = 0; i < N; i++) {
        if (do_fill) {
            fill_store();
            blockmix_r1<MW, DR_UNROLL>(lo_f, hi_f);
        }
        if (do_mix) {
            cp_async_wait_all();
            __syncwarp();
            uint32_t vlo[16], vhi[16];
#pragma unroll
            for (int k = 0; k < 8; k++) set_chunk(vlo, vhi, k, lds128(own_m + ((k ^ swz) << 4)));
            __syncwarp();
            blockmix_r1_xor<MW, DR_UNROLL>(lo_m, hi_m, vlo, vhi);
            if (i + 1 < N) mix_prefetch();
        }
    }
#undef MIX_PREFETCH_K
#undef FILL_STORE_K
    if (do_fill) {
#pragma unroll
        for (int k = 0; k < 8; k++) p.Xfill[(size_t)k * p.x_stride + slot] = ROW_CHUNK(lo_f, hi_f, k);
    }
    if (do_mix) {
#pragma unroll
        for (int k = 0; k < 8; k++) p.Xmix[(size_t)k * p.x_stride + slot] = ROW_CHUNK(lo_m, hi_m, k);
    }
    if (p.cta_trace && threadIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        p.cta_trace[3 * (size_t)blockIdx.x + 1] = t;
    }
}

// =================================================================================================
// K2f: phased ROMix.  Every thread runs TWO labels of the same layer, A = slot t and B = slot t + S
// (S = p.pair_offset, the engine's resident slot count), with the slot's two scratchpads: first N fill steps of both, then N
// mix steps of both.  So a whole launch first only writes the scratchpads and then only reads them,
// and HBM stops turning its bus around between reads and writes in every step (DESIGN.md §4).
// In the mix loop each label's dependent row read is requested with cp.async while the other label's
// BlockMix runs, the same window romix_pipe_kernel gives its mix read.  A warp of a partial layer whose
// B slots lie past n_slots runs A alone (fill, then mix); a layer of at most S labels has no B at all, so
// it keeps one label per thread and as many threads as the pipelined kernel would give it.  One launch is a whole layer: no state crosses
// launches.
// The step loops hold little besides the BlockMix arithmetic, because the ALU pipe sets the fill phase's pace:
//  - fill: the lanes write their rows into the warp's 4 KiB tile, whose byte order is the scratchpad row's, and lane 0
//    sends the tile to HBM with one TMA bulk store.  Tiles are double-buffered per label (single at 512 threads, where
//    two would not fit in shared memory), so a step waits only on the store issued two steps earlier.
//  - mix: the 32 row indices pass through shared memory instead of 8 shuffles: each lane stores its j, then reads the
//    8 it needs for its transposed cp.async requests (4 whole 128-B lines each) with two 16-byte loads.
// Shared memory per warp: PHASED_BUFS(TPB) x (tile A, tile B), then 2 x 128 B of row indices.
// =================================================================================================
#define PHASED_BUFS(tpb) ((tpb) <= 256 ? 2u : 1u)
#define PHASED_WARP_SMEM(tpb) (PHASED_BUFS(tpb) * 8192u + 256u)

__device__ __forceinline__ void sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
// bulk_s2g to the 64-bit address {lo, hi}, issued by the lanes with `issue` set, without a branch around it
__device__ __forceinline__ void bulk_s2g_lohi_if(bool issue, uint32_t lo, uint32_t hi, uint32_t src_smem, uint32_t bytes) {
    asm volatile("{\n\t.reg .pred p;\n\t.reg .b64 a;\n\tsetp.ne.u32 p, %4, 0;\n\tmov.b64 a, {%0, %1};\n\t"
                 "@p cp.async.bulk.global.shared::cta.bulk_group [a], [%2], %3;\n\t}"
                 ::"r"(lo), "r"(hi), "r"(src_smem), "r"(bytes), "r"((uint32_t)issue) : "memory");
}

template <int MW, int TPB>
__global__ void __launch_bounds__(TPB) romix_phased_kernel(const RomixParams p) {
    constexpr int DR = 4;
    constexpr uint32_t BUFS = PHASED_BUFS(TPB);
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const uint32_t T = p.pair_offset;
    const uint32_t slot = blockIdx.x * TPB + threadIdx.x;
    if (slot >= T || slot >= p.n_slots) return;     // both are multiples of 32: whole warps leave together
    const bool has_b = slot + T < p.n_slots;        // warp-uniform
    const uint32_t lane = threadIdx.x & 31, warp_in_cta = threadIdx.x >> 5;
    const uint32_t N = p.N, mask = N - 1;
    const uint32_t tile_a = smem_u32(smem_raw) + warp_in_cta * PHASED_WARP_SMEM(TPB), tile_b = tile_a + 4096;
    const uint32_t idx_a = tile_a + BUFS * 8192, idx_b = idx_a + 128;
    const uint32_t own_a = tile_a + lane * 128, own_b = tile_b + lane * 128;
    const uint32_t swz = lane & 7, tr_row = lane >> 3, tr_c = lane & 7;
    const uint32_t tile_a_tr = tile_a + tr_row * 128 + (tr_c << 4), tile_b_tr = tile_b + tr_row * 128 + (tr_c << 4);
    // lane s's row index sits at word (s & 3) * 8 + (s >> 2); lane t's k-th transposed request needs lane 4k + (t >> 3),
    // so its 8 indices are the words tr_row * 8 .. tr_row * 8 + 7
    const uint32_t idx_put = ((lane & 3) * 8 + (lane >> 2)) * 4, idx_get = tr_row * 32;
    const size_t warp = slot >> 5;
    uint4 *const va = p.V + (warp * 2) * (size_t)N * 256, *const vb = va + (size_t)N * 256;   // row i at + i * 256
    // this lane's base in the warp's two scratchpad regions as {lo, hi} (see romix_pipe_kernel): `hi` is constant
    // within a region
    const uint64_t va64 = (uint64_t)(va + lane), vb64 = (uint64_t)(vb + lane);
    const uint32_t va_lo = (uint32_t)va64, va_hi = (uint32_t)(va64 >> 32);
    const uint32_t vb_lo = (uint32_t)vb64, vb_hi = (uint32_t)(vb64 >> 32);
    const bool issuer = lane == 0;
    uint32_t ra = (uint32_t)(uint64_t)va, rb = (uint32_t)(uint64_t)vb;   // low word of row i's address; +4096 per step

    uint32_t lo_a[16], hi_a[16], lo_b[16], hi_b[16];
#pragma unroll
    for (int k = 0; k < 8; k++) set_chunk(lo_a, hi_a, k, p.X[(size_t)k * p.x_stride + slot]);
    if (has_b) {
#pragma unroll
        for (int k = 0; k < 8; k++) set_chunk(lo_b, hi_b, k, p.X[(size_t)k * p.x_stride + slot + T]);
    }

    // before a tile is rewritten, the bulk store that last read it has read it (the issuing lane waits; the
    // __syncwarp after the wait holds the others back)
#define TILE_FREE()                                                    \
    {                                                                  \
        if (BUFS == 2) bulk_wait_read<1>(); else bulk_wait_read<0>(); \
        __syncwarp();                                                  \
    }
    // own row -> tile (swizzled: chunk k at position k ^ (lane & 7), which is where the scratchpad row keeps it)
#define ROW_TO_TILE(own, lo, hi) \
    _Pragma("unroll") for (int k = 0; k < 8; k++) sts128(own + ((k ^ swz) << 4), ROW_CHUNK(lo, hi, k));
    // request row V[Integerify(hi)] of every lane's label into the tile: 8 x (4 rows x 128 B) per warp
#define ROW_REQUEST_K(tile_tr, jv, vlo, vhi, k) cp_async16_lohi<(k) * 512>(tile_tr + (k) * 512, mad_u32(jv, 4096u, vlo), vhi);
#define ROW_REQUEST(tile_tr, idx, hi, vlo, vhi)                                                                    \
    {                                                                                                              \
        sts32(idx + idx_put, hi[0] & mask);                                                                        \
        __syncwarp();                                                                                              \
        const uint4 j0 = lds128(idx + idx_get), j1 = lds128(idx + idx_get + 16);                                   \
        ROW_REQUEST_K(tile_tr, j0.x, vlo, vhi, 0) ROW_REQUEST_K(tile_tr, j0.y, vlo, vhi, 1)                        \
        ROW_REQUEST_K(tile_tr, j0.z, vlo, vhi, 2) ROW_REQUEST_K(tile_tr, j0.w, vlo, vhi, 3)                        \
        ROW_REQUEST_K(tile_tr, j1.x, vlo, vhi, 4) ROW_REQUEST_K(tile_tr, j1.y, vlo, vhi, 5)                        \
        ROW_REQUEST_K(tile_tr, j1.z, vlo, vhi, 6) ROW_REQUEST_K(tile_tr, j1.w, vlo, vhi, 7)                        \
        cp_async_commit();                                                                                         \
    }
    // the lane's landed row out of the tile, then X <- BlockMix(X ^ row)
#define MIX_FROM_TILE(own, lo, hi)                                                                       \
    {                                                                                                    \
        uint32_t vlo[16], vhi[16];                                                                       \
        _Pragma("unroll") for (int k = 0; k < 8; k++) set_chunk(vlo, vhi, k, lds128(own + ((k ^ swz) << 4))); \
        __syncwarp();                                                                                    \
        blockmix_r1_xor<MW, DR>(lo, hi, vlo, vhi);                                                       \
    }

    uint32_t buf = 0;   // byte offset of this step's tile pair: 0 or 8192
    if (has_b) {
        for (uint32_t i = 0; i < N; i++) {
            TILE_FREE()
            ROW_TO_TILE(own_a + buf, lo_a, hi_a)
            ROW_TO_TILE(own_b + buf, lo_b, hi_b)
            fence_proxy_async_smem();
            __syncwarp();
            bulk_s2g_lohi_if(issuer, ra, va_hi, tile_a + buf, 4096);
            bulk_s2g_lohi_if(issuer, rb, vb_hi, tile_b + buf, 4096);
            bulk_commit();
            ra = mad_u32(1u, 4096u, ra); rb = mad_u32(1u, 4096u, rb);
            buf ^= (BUFS - 1) * 8192;
            blockmix_r1_x2<MW, DR>(lo_a, hi_a, lo_b, hi_b);
        }
    } else {
        for (uint32_t i = 0; i < N; i++) {
            TILE_FREE()
            ROW_TO_TILE(own_a + buf, lo_a, hi_a)
            fence_proxy_async_smem();
            __syncwarp();
            bulk_s2g_lohi_if(issuer, ra, va_hi, tile_a + buf, 4096);
            bulk_commit();
            ra = mad_u32(1u, 4096u, ra);
            buf ^= (BUFS - 1) * 8192;
            blockmix_r1<MW, DR>(lo_a, hi_a);
        }
    }
    // every row is in HBM before any lane requests one, and no store still reads a tile the requests land in
    bulk_wait_all<0>();
    __syncwarp();
#ifndef B200POST_PHASED_FILL_ONLY   // a scratch build of tools/romix_phase_split.py times the fill phase alone
    if (has_b) {
        ROW_REQUEST(tile_b_tr, idx_b, hi_b, vb_lo, vb_hi)
        for (uint32_t i = 0; i + 1 < N; i++) {
            ROW_REQUEST(tile_a_tr, idx_a, hi_a, va_lo, va_hi)
            asm volatile("cp.async.wait_group 1;" ::: "memory");   // B's row has landed; A's is in flight
            __syncwarp();
            MIX_FROM_TILE(own_b, lo_b, hi_b)
            ROW_REQUEST(tile_b_tr, idx_b, hi_b, vb_lo, vb_hi)
            asm volatile("cp.async.wait_group 1;" ::: "memory");
            __syncwarp();
            MIX_FROM_TILE(own_a, lo_a, hi_a)
        }
        // the last step: no further request of B
        ROW_REQUEST(tile_a_tr, idx_a, hi_a, va_lo, va_hi)
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncwarp();
        MIX_FROM_TILE(own_b, lo_b, hi_b)
        cp_async_wait_all();
        __syncwarp();
        MIX_FROM_TILE(own_a, lo_a, hi_a)
    } else {
        for (uint32_t i = 0; i < N; i++) {
            ROW_REQUEST(tile_a_tr, idx_a, hi_a, va_lo, va_hi)
            cp_async_wait_all();
            __syncwarp();
            MIX_FROM_TILE(own_a, lo_a, hi_a)
        }
    }
#endif
#undef TILE_FREE
#undef ROW_TO_TILE
#undef ROW_REQUEST_K
#undef ROW_REQUEST
#undef MIX_FROM_TILE
#pragma unroll
    for (int k = 0; k < 8; k++) p.X[(size_t)k * p.x_stride + slot] = ROW_CHUNK(lo_a, hi_a, k);
    if (has_b) {
#pragma unroll
        for (int k = 0; k < 8; k++) p.X[(size_t)k * p.x_stride + slot + T] = ROW_CHUNK(lo_b, hi_b, k);
    }
}

// =================================================================================================
// K3: PBKDF2 final + label output (TMA bulk store) + VRF candidate per CTA
// =================================================================================================
constexpr int FINAL_TPB = 128;

// warp arg-min of (best, best_i) over the lanes with has != 0, by shuffles; every lane ends with the warp's winner
__device__ __forceinline__ void warp_argmin(uint32_t (&best)[8], uint64_t &best_i, uint32_t &has) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        uint32_t o[8];
#pragma unroll
        for (int k = 0; k < 8; k++) o[k] = __shfl_xor_sync(0xffffffffu, best[k], off);
        const uint64_t oi = __shfl_xor_sync(0xffffffffu, best_i, off);
        const uint32_t oh = __shfl_xor_sync(0xffffffffu, has, off);
        const bool take = oh && (!has || cand_less(o, oi, best, best_i));
        if (take) {
#pragma unroll
            for (int k = 0; k < 8; k++) best[k] = o[k];
            best_i = oi; has = 1;
        }
    }
}

// VRF nonce candidate of one CTA: min over valid slots with label32 < difficulty (strict), lowest index on ties.
// Block-wide: every thread of the CTA calls it.
__device__ __forceinline__ void cta_vrf_candidate(bool valid, const uint32_t (&lab)[8], uint64_t index,
                                                  const uint32_t *__restrict__ vrf_be, VrfCandidate *warp_best,
                                                  VrfCandidate *__restrict__ cta_cand) {
    uint32_t diff[8];
#pragma unroll
    for (int k = 0; k < 8; k++) diff[k] = vrf_be[k];
    // cand_less with equal labels compares indices 0 < 0 = false => strict '<' on the label
    const bool cand = valid && cand_less(lab, 0, diff, 0);
    if (!__syncthreads_or(cand)) {
        if (threadIdx.x == 0) cta_cand[blockIdx.x].found = 0;
        return;
    }
    // rare path: warp argmin by shuffles, then thread 0 merges the per-warp winners
    uint32_t best[8];
    uint64_t best_i = index;
    uint32_t has = cand ? 1u : 0u;
#pragma unroll
    for (int k = 0; k < 8; k++) best[k] = lab[k];
    warp_argmin(best, best_i, has);
    if ((threadIdx.x & 31) == 0) {
        VrfCandidate &w = warp_best[threadIdx.x >> 5];
#pragma unroll
        for (int k = 0; k < 8; k++) w.label_be[k] = best[k];
        w.index = best_i; w.found = has; w.pad = 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        VrfCandidate r = warp_best[0];
        for (int wv = 1; wv < FINAL_TPB / 32; wv++) {
            const VrfCandidate c = warp_best[wv];
            if (c.found && (!r.found || cand_less(c.label_be, c.index, r.label_be, r.index))) r = c;
        }
        cta_cand[blockIdx.x] = r;
    }
}

__global__ void __launch_bounds__(FINAL_TPB) pbkdf2_final_kernel(LabelJob job, const uint4 *__restrict__ X, uint32_t x_stride,
                                                                 uint32_t n_slots, uint8_t *__restrict__ out16,
                                                                 const uint32_t *__restrict__ vrf_be,
                                                                 VrfCandidate *__restrict__ cta_cand) {
    __shared__ __align__(128) uint4 stage[FINAL_TPB];
    __shared__ VrfCandidate warp_best[FINAL_TPB / 32];
    const uint32_t slot = blockIdx.x * FINAL_TPB + threadIdx.x;
    const bool valid = slot < job.n_valid;
    uint32_t lab[8];
    uint64_t index = 0;
    if (slot < n_slots) {
        uint32_t c[8];
        load_commit(job, valid ? slot : 0, c);
        uint32_t lo[16], hi[16];
#pragma unroll
        for (int k = 0; k < 8; k++) set_chunk(lo, hi, k, X[(size_t)k * x_stride + slot]);
        index = slot_index(job, slot);
        label_final(c, index, lo, hi, lab);
    } else {
#pragma unroll
        for (int k = 0; k < 8; k++) lab[k] = 0xffffffffu;
    }
    // label = first 16 of the 32 output bytes; bytes are the big-endian serialisation of lab[]
    stage[threadIdx.x] = make_uint4(bswap32(lab[0]), bswap32(lab[1]), bswap32(lab[2]), bswap32(lab[3]));
    fence_proxy_async_smem();
    __syncthreads();
    const uint32_t cta_first = blockIdx.x * FINAL_TPB;
    if (threadIdx.x == 0 && cta_first < job.n_valid) {
        const uint32_t n_here = min((uint32_t)FINAL_TPB, job.n_valid - cta_first);
        // one TMA bulk store per CTA: n_here x 16 contiguous bytes (16-B aligned, multiple of 16)
        bulk_s2g(out16 + (size_t)cta_first * 16, smem_u32(stage), n_here * 16);
        bulk_commit();
        bulk_wait_all<0>();
    }
    if (vrf_be == nullptr) return;
    cta_vrf_candidate(valid, lab, index, vrf_be, warp_best, cta_cand);
}

// K3w: K3's label with all 32 bytes kept, for gathers whose items need the whole label32 (VRF-nonce checks).  Bytes
// 0-15 go to out16 exactly as K3 stores them, bytes 16-31 to out_hi16 at the same item position; each half leaves by
// its own TMA bulk store.  No VRF-candidate path: a gather has none.
__global__ void __launch_bounds__(FINAL_TPB) pbkdf2_final_wide_kernel(LabelJob job, const uint4 *__restrict__ X, uint32_t x_stride,
                                                                      uint32_t n_slots, uint8_t *__restrict__ out16,
                                                                      uint8_t *__restrict__ out_hi16) {
    __shared__ __align__(128) uint4 stage_lo[FINAL_TPB];
    __shared__ __align__(128) uint4 stage_hi[FINAL_TPB];
    const uint32_t slot = blockIdx.x * FINAL_TPB + threadIdx.x;
    const bool valid = slot < job.n_valid;
    uint32_t lab[8];
    if (slot < n_slots) {
        uint32_t c[8];
        load_commit(job, valid ? slot : 0, c);
        uint32_t lo[16], hi[16];
#pragma unroll
        for (int k = 0; k < 8; k++) set_chunk(lo, hi, k, X[(size_t)k * x_stride + slot]);
        label_final(c, slot_index(job, slot), lo, hi, lab);
    } else {
#pragma unroll
        for (int k = 0; k < 8; k++) lab[k] = 0xffffffffu;
    }
    stage_lo[threadIdx.x] = make_uint4(bswap32(lab[0]), bswap32(lab[1]), bswap32(lab[2]), bswap32(lab[3]));
    stage_hi[threadIdx.x] = make_uint4(bswap32(lab[4]), bswap32(lab[5]), bswap32(lab[6]), bswap32(lab[7]));
    fence_proxy_async_smem();
    __syncthreads();
    const uint32_t cta_first = blockIdx.x * FINAL_TPB;
    if (threadIdx.x == 0 && cta_first < job.n_valid) {
        const uint32_t n_here = min((uint32_t)FINAL_TPB, job.n_valid - cta_first);
        bulk_s2g(out16 + (size_t)cta_first * 16, smem_u32(stage_lo), n_here * 16);
        bulk_s2g(out_hi16 + (size_t)cta_first * 16, smem_u32(stage_hi), n_here * 16);
        bulk_commit();
        bulk_wait_all<0>();
    }
}

// K3c: K3's label, compared with the expected 16 bytes instead of stored (checking stored POST data).  The CTA's
// expected labels arrive by one TMA bulk load issued before the PBKDF2, so the load overlaps its Keccak-f work.
// Each warp writes one ballot word of mismatching slots to mismatch_bits[slot / 32] (n_slots / 32 words, all
// written) and adds its popcount to *mismatch_count only when it is non-zero.  VRF candidates as in K3.
__global__ void __launch_bounds__(FINAL_TPB) pbkdf2_final_compare_kernel(LabelJob job, const uint4 *__restrict__ X, uint32_t x_stride,
                                                                         uint32_t n_slots, const uint8_t *__restrict__ expect16,
                                                                         uint32_t *__restrict__ mismatch_bits,
                                                                         uint32_t *__restrict__ mismatch_count,
                                                                         const uint32_t *__restrict__ vrf_be,
                                                                         VrfCandidate *__restrict__ cta_cand) {
    __shared__ __align__(128) uint4 expect[FINAL_TPB];
    __shared__ __align__(8) uint64_t bar_storage;
    __shared__ VrfCandidate warp_best[FINAL_TPB / 32];
    const uint32_t cta_first = blockIdx.x * FINAL_TPB;
    const uint32_t slot = cta_first + threadIdx.x;
    const bool valid = slot < job.n_valid;
    const bool any_valid = cta_first < job.n_valid;
    const uint32_t bar = smem_u32(&bar_storage);
    if (threadIdx.x == 0 && any_valid) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const uint32_t n_here = min((uint32_t)FINAL_TPB, job.n_valid - cta_first);
        mbar_expect_tx(bar, n_here * 16);
        bulk_g2s(smem_u32(expect), expect16 + (size_t)cta_first * 16, n_here * 16, bar);
    }
    uint32_t lab[8];
    uint64_t index = 0;
    if (slot < n_slots) {
        uint32_t c[8];
        load_commit(job, valid ? slot : 0, c);
        uint32_t lo[16], hi[16];
#pragma unroll
        for (int k = 0; k < 8; k++) set_chunk(lo, hi, k, X[(size_t)k * x_stride + slot]);
        index = slot_index(job, slot);
        label_final(c, index, lo, hi, lab);
    } else {
#pragma unroll
        for (int k = 0; k < 8; k++) lab[k] = 0xffffffffu;
    }
    __syncthreads();   // the barrier is initialised before anyone waits on it
    bool bad = false;
    if (any_valid) {
        mbar_wait(bar, 0);
        if (valid) {
            const uint4 e = expect[threadIdx.x];
            bad = (e.x != bswap32(lab[0])) | (e.y != bswap32(lab[1])) | (e.z != bswap32(lab[2])) | (e.w != bswap32(lab[3]));
        }
    }
    const uint32_t ballot = __ballot_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0 && slot < n_slots) {
        mismatch_bits[slot >> 5] = ballot;
        if (ballot) atomicAdd(mismatch_count, (uint32_t)__popc(ballot));
    }
    if (vrf_be == nullptr) return;
    cta_vrf_candidate(valid, lab, index, vrf_be, warp_best, cta_cand);
}

// K4: merge the per-CTA candidates of one wave into the running minimum (1 CTA, 256 threads)
__global__ void __launch_bounds__(256) vrf_merge_kernel(const VrfCandidate *__restrict__ cta_cand, uint32_t n_cta,
                                                         VrfCandidate *__restrict__ running) {
    __shared__ VrfCandidate sh[256];
    VrfCandidate r;
    r.found = 0; r.index = 0; r.pad = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) r.label_be[k] = 0xffffffffu;
    for (uint32_t i = threadIdx.x; i < n_cta; i += 256) {
        const VrfCandidate c = cta_cand[i];
        if (c.found && (!r.found || cand_less(c.label_be, c.index, r.label_be, r.index))) r = c;
    }
    sh[threadIdx.x] = r;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
            const VrfCandidate c = sh[threadIdx.x + s];
            VrfCandidate &m = sh[threadIdx.x];
            if (c.found && (!m.found || cand_less(c.label_be, c.index, m.label_be, m.index))) m = c;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const VrfCandidate c = sh[0];
        VrfCandidate m = *running;
        if (c.found && (!m.found || cand_less(c.label_be, c.index, m.label_be, m.index))) *running = c;
    }
}

// =================================================================================================
// launch table
// =================================================================================================
cudaError_t launch_pbkdf2_expand(const LabelJob &job, uint4 *X, uint32_t x_stride, uint32_t n_slots, cudaStream_t s) {
    if (n_slots == 0) return cudaSuccess;
    pbkdf2_expand_kernel<<<(n_slots + 127) / 128, 128, 0, s>>>(job, X, x_stride, n_slots);
    return cudaGetLastError();
}

uint32_t pbkdf2_final_ctas(uint32_t n_slots) { return (n_slots + FINAL_TPB - 1) / FINAL_TPB; }

cudaError_t launch_pbkdf2_final_compare(const LabelJob &job, const uint4 *X, uint32_t x_stride, uint32_t n_slots,
                                        const uint8_t *expect16, uint32_t *mismatch_bits, uint32_t *mismatch_count,
                                        const uint32_t *vrf_difficulty_be, VrfCandidate *cta_cand, cudaStream_t s) {
    if (n_slots == 0) return cudaSuccess;
    pbkdf2_final_compare_kernel<<<pbkdf2_final_ctas(n_slots), FINAL_TPB, 0, s>>>(job, X, x_stride, n_slots, expect16, mismatch_bits,
                                                                                 mismatch_count, vrf_difficulty_be, cta_cand);
    return cudaGetLastError();
}

cudaError_t launch_pbkdf2_final(const LabelJob &job, const uint4 *X, uint32_t x_stride, uint32_t n_slots, uint8_t *out16,
                                const uint32_t *vrf_difficulty_be, VrfCandidate *cta_cand, cudaStream_t s) {
    if (n_slots == 0) return cudaSuccess;
    pbkdf2_final_kernel<<<pbkdf2_final_ctas(n_slots), FINAL_TPB, 0, s>>>(job, X, x_stride, n_slots, out16,
                                                                         vrf_difficulty_be, cta_cand);
    return cudaGetLastError();
}

cudaError_t launch_pbkdf2_final_wide(const LabelJob &job, const uint4 *X, uint32_t x_stride, uint32_t n_slots, uint8_t *out16,
                                     uint8_t *out_hi16, cudaStream_t s) {
    if (n_slots == 0) return cudaSuccess;
    pbkdf2_final_wide_kernel<<<pbkdf2_final_ctas(n_slots), FINAL_TPB, 0, s>>>(job, X, x_stride, n_slots, out16, out_hi16);
    return cudaGetLastError();
}

cudaError_t launch_vrf_merge(const VrfCandidate *cta_cand, uint32_t n_cta, VrfCandidate *running, cudaStream_t s) {
    vrf_merge_kernel<<<1, 256, 0, s>>>(cta_cand, n_cta, running);
    return cudaGetLastError();
}

size_t romix_smem_bytes(int variant, int tpb) {
    const size_t warps = (size_t)tpb / 32;
    if (variant == ROMIX_COALESCED) return warps * 4096;
    if (variant == ROMIX_BULK) return warps * 8192 + warps * 8;
    if (variant == ROMIX_PIPELINED) return warps * 8192;
    if (variant == ROMIX_PHASED) return warps * PHASED_WARP_SMEM(tpb);
    return 0;
}

const char *romix_variant_name(int variant) {
    switch (variant) {
        case ROMIX_DIRECT: return "direct";
        case ROMIX_COALESCED: return "coalesced";
        case ROMIX_BULK: return "bulk";
        case ROMIX_NOMEM: return "nomem";
        case ROMIX_PIPELINED: return "pipelined";
        case ROMIX_PHASED: return "phased";
    }
    return "?";
}

typedef void (*romix_fn)(const RomixParams);
typedef void (*pipe_fn)(const PipeParams);

// rotate-form masks compiled in (see chacha20_8): 0 = all funnel shifts, 1 = the 16- and 8-bit rotates as PRMT
#define B200POST_MW_LIST(X) X(0) X(1)

template <int VARIANT, int MW>
static romix_fn pick_tpb(int tpb) {
    switch (tpb) {
        case 128: return romix_kernel<VARIANT, MW, 128>;
        case 256: return romix_kernel<VARIANT, MW, 256>;
    }
    return nullptr;
}
template <int VARIANT>
static romix_fn pick_mw(int mw, int tpb) {
    switch (mw) {
#define X(m) case m: return pick_tpb<VARIANT, m>(tpb);
        B200POST_MW_LIST(X)
#undef X
    }
    return nullptr;
}
static romix_fn pick(int variant, int mw, int tpb) {
    switch (variant) {
        case ROMIX_DIRECT: return pick_mw<ROMIX_DIRECT>(mw, tpb);
        case ROMIX_COALESCED: return pick_mw<ROMIX_COALESCED>(mw, tpb);
        case ROMIX_BULK: return pick_mw<ROMIX_BULK>(mw, tpb);
        case ROMIX_NOMEM: return pick_mw<ROMIX_NOMEM>(mw, tpb);
    }
    return nullptr;
}
template <int MW>
static pipe_fn pick_pipe_tpb(int tpb, int dr_unroll) {
    if (dr_unroll == 4) {
        switch (tpb) {
            case 64: return romix_pipe_kernel<MW, 64, 4>;
            case 128: return romix_pipe_kernel<MW, 128, 4>;
            case 256: return romix_pipe_kernel<MW, 256, 4>;
            case 512: return romix_pipe_kernel<MW, 512, 4>;
        }
    } else {
        switch (tpb) {
            case 64: return romix_pipe_kernel<MW, 64, 1>;
            case 128: return romix_pipe_kernel<MW, 128, 1>;
            case 256: return romix_pipe_kernel<MW, 256, 1>;
            case 512: return romix_pipe_kernel<MW, 512, 1>;
        }
    }
    return nullptr;
}
static pipe_fn pick_pipe(int mw, int tpb, int dr_unroll) {
    switch (mw) {
#define X(m) case m: return pick_pipe_tpb<m>(tpb, dr_unroll);
        B200POST_MW_LIST(X)
#undef X
    }
    return nullptr;
}

template <int MW>
static romix_fn pick_phased_tpb(int tpb) {
    switch (tpb) {
        case 64: return romix_phased_kernel<MW, 64>;
        case 128: return romix_phased_kernel<MW, 128>;
        case 256: return romix_phased_kernel<MW, 256>;
        case 512: return romix_phased_kernel<MW, 512>;
    }
    return nullptr;
}
static romix_fn pick_phased(int mw, int tpb) {
    switch (mw) {
#define X(m) case m: return pick_phased_tpb<m>(tpb);
        B200POST_MW_LIST(X)
#undef X
    }
    return nullptr;
}

bool romix_mask_supported(int mw) {
    switch (mw) {
#define X(m) case m: return true;
        B200POST_MW_LIST(X)
#undef X
    }
    return false;
}

int romix_max_ctas_per_sm(int variant, int rot_mask, int tpb, int dr_unroll) {
    const size_t smem = romix_smem_bytes(variant, tpb);
    int n = 0;
    if (variant == ROMIX_PIPELINED) {
        pipe_fn fn = pick_pipe(rot_mask, tpb, dr_unroll);
        if (!fn) return 0;
        if (smem > 48 * 1024) cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, tpb, smem) != cudaSuccess) return 0;
        return n;
    }
    romix_fn fn = variant == ROMIX_PHASED ? pick_phased(rot_mask, tpb) : pick(variant, rot_mask, tpb);
    if (!fn) return 0;
    if (smem > 48 * 1024) cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, tpb, smem) != cudaSuccess) return 0;
    return n;
}

cudaError_t launch_romix(int variant, int rot_mask, int tpb, const RomixParams &p, cudaStream_t s) {
    if (p.n_slots == 0) return cudaSuccess;
    const bool phased = variant == ROMIX_PHASED;
    romix_fn fn = phased ? pick_phased(rot_mask, tpb) : pick(variant, rot_mask, tpb);
    if (!fn) return cudaErrorInvalidValue;
    const size_t smem = romix_smem_bytes(variant, tpb);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    if (phased && (p.pair_offset % 32 || 2 * (uint64_t)p.pair_offset < p.n_slots)) return cudaErrorInvalidValue;
    const uint32_t threads = phased && p.pair_offset < p.n_slots ? p.pair_offset : p.n_slots;
    fn<<<(threads + tpb - 1) / tpb, tpb, smem, s>>>(p);
    return cudaGetLastError();
}

uint32_t romix_lowlat_warps(uint32_t n_slots, int sm_count) {
    const uint32_t full = (uint32_t)sm_count * 4;             // one warp per scheduler slot
    return n_slots < full ? (n_slots ? n_slots : 1) : full;
}
cudaError_t launch_romix_lowlat(int rot_mask, const RomixParams &p, uint32_t n_warps, cudaStream_t s) {
    if (p.n_slots == 0) return cudaSuccess;
    if (n_warps == 0 || (uint64_t)n_warps * 32 < p.n_slots) return cudaErrorInvalidValue;
    if (rot_mask == 1) romix_lowlat_kernel<1><<<n_warps, 32, 0, s>>>(p, n_warps);
    else romix_lowlat_kernel<0><<<n_warps, 32, 0, s>>>(p, n_warps);
    return cudaGetLastError();
}

cudaError_t launch_romix_pipe(int rot_mask, int tpb, int dr_unroll, const PipeParams &p, cudaStream_t s) {
    const uint32_t n = p.n_fill > p.n_mix ? p.n_fill : p.n_mix;
    if (n == 0) return cudaSuccess;
    pipe_fn fn = pick_pipe(rot_mask, tpb, dr_unroll);
    if (!fn) return cudaErrorInvalidValue;
    const size_t smem = romix_smem_bytes(ROMIX_PIPELINED, tpb);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    fn<<<(n + tpb - 1) / tpb, tpb, smem, s>>>(p);
    return cudaGetLastError();
}

}  // namespace b200post
