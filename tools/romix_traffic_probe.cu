// tools/romix_traffic_probe.cu — dev probe: does HBM move the pipelined ROMix layer's traffic faster when a launch
// writes every scratchpad first and reads them afterwards, instead of writing and reading in every step?
//
// It replays the memory traffic of `romix_pipe_kernel` with no ChaCha: one slot per thread, 256-thread CTAs, two
// N x 4 KiB regions per warp (the engine's per-warp scratchpad layout), 128-byte rows written through the same
// swizzled 4 KiB shared-memory tile as 8 x 512 B `st.global.cs`, and random rows read by the same transposed
// 8 x 16 B `cp.async` per lane.  A row index depends on the row read before it, as Integerify does.
//   (a) interleaved: per step, one row store into region 0 and one random row read from region 1 per warp, the read
//       requested at the end of the previous step and waited for after the store (romix_pipe_kernel's schedule);
//   (b) phased: N steps of two row stores per warp (regions 0 and 1), then N steps of two random row reads per warp,
//       each read requested while the other label's row is consumed (the schedule of a two-labels-per-thread layer).
// Both move 2 x 128 x N bytes per label; (b) runs two labels per thread, so it moves twice the bytes per launch.
// The timed launches alternate a, b, a, b, ...; each prints one JSON line.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/romix_traffic_probe tools/romix_traffic_probe.cu
// Run:   tools/romix_traffic_probe [N=8192] [slots=SMs x 256] [pairs=3]
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <utility>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("{\"error\": \"%s: %s\"}\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

constexpr int TPB = 256;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void st_stream(uint4 *p, const uint4 &v) {
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N_PENDING>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N_PENDING) : "memory"); }
__device__ __forceinline__ void sts128(uint32_t a, const uint4 &v) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}

struct Warp {
    uint32_t lane, swz, tr_row, tr_c;
    uint32_t tile[2];   // two 4 KiB tiles of this warp
    uint4 *region[2];   // this lane's column (+ lane) of the warp's two N x 4 KiB regions
};

// write row i of one label: own row -> tile (swizzled), tile -> HBM as 8 x 512 contiguous bytes per warp
__device__ __forceinline__ void row_store(const Warp &w, int t, uint4 *region, uint32_t i, uint32_t x) {
    const uint32_t own = w.tile[t] + w.lane * 128;
#pragma unroll
    for (int k = 0; k < 8; k++) sts128(own + ((k ^ w.swz) << 4), make_uint4(x + k, i, w.lane, k));
    __syncwarp();
#pragma unroll
    for (int k = 0; k < 8; k++) st_stream(region + (size_t)i * 256 + k * 32, lds128(w.tile[t] + (k * 4 + w.tr_row) * 128 + (w.tr_c << 4)));
    __syncwarp();
}
// request row j (per lane) of one label into its tile: 8 x (4 rows x 128 B) per warp
__device__ __forceinline__ void row_request(const Warp &w, int t, const uint4 *region, uint32_t j) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint32_t jr = __shfl_sync(0xffffffffu, j, k * 4 + w.tr_row);
        cp_async16(w.tile[t] + (k * 4 + w.tr_row) * 128 + (w.tr_c << 4), region + (size_t)jr * 256 + k * 32);
    }
    cp_async_commit();
}
// read this lane's landed row back from the tile and derive the next row index from it
__device__ __forceinline__ uint32_t row_consume(const Warp &w, int t, uint32_t j, uint32_t mask) {
    const uint32_t own = w.tile[t] + w.lane * 128;
    uint32_t acc = j * 0x9E3779B9u;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint4 v = lds128(own + ((k ^ w.swz) << 4));
        acc = (acc ^ v.x ^ v.y ^ v.z ^ v.w) * 0x85EBCA6Bu + k;
    }
    return (acc ^ (acc >> 15)) & mask;
}

template <bool PHASED>
__global__ void __launch_bounds__(TPB) traffic(uint4 *V, uint32_t N, uint32_t n_slots, uint32_t *sink) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const uint32_t slot = blockIdx.x * TPB + threadIdx.x;
    if (slot >= n_slots) return;   // n_slots is a multiple of 32
    Warp w;
    w.lane = threadIdx.x & 31; w.swz = w.lane & 7; w.tr_row = w.lane >> 3; w.tr_c = w.lane & 7;
    w.tile[0] = smem_u32(smem_raw) + (threadIdx.x >> 5) * 8192; w.tile[1] = w.tile[0] + 4096;
    const size_t warp = slot >> 5;
    // the lane's column of row 0; row r of its transposed copy k is at + r * 256 + k * 32
    w.region[0] = V + (warp * 2) * (size_t)N * 256 + w.lane;
    w.region[1] = V + (warp * 2 + 1) * (size_t)N * 256 + w.lane;
    const uint32_t mask = N - 1;
    uint32_t ja = (slot * 2654435761u) & mask, jb = (slot * 40503u + 7) & mask;
    if (!PHASED) {
        row_request(w, 1, w.region[1], jb);
        for (uint32_t i = 0; i < N; i++) {
            row_store(w, 0, w.region[0], i, ja);
            cp_async_wait<0>();
            __syncwarp();
            jb = row_consume(w, 1, jb, mask);
            __syncwarp();
            if (i + 1 < N) row_request(w, 1, w.region[1], jb);
        }
    } else {
        for (uint32_t i = 0; i < N; i++) {
            row_store(w, 0, w.region[0], i, ja);
            row_store(w, 1, w.region[1], i, jb);
        }
        row_request(w, 1, w.region[1], jb);
        for (uint32_t i = 0; i < N; i++) {
            row_request(w, 0, w.region[0], ja);
            cp_async_wait<1>();   // B's row has landed; A's is in flight
            __syncwarp();
            jb = row_consume(w, 1, jb, mask);
            __syncwarp();
            if (i + 1 < N) { row_request(w, 1, w.region[1], jb); cp_async_wait<1>(); }
            else cp_async_wait<0>();
            __syncwarp();
            ja = row_consume(w, 0, ja, mask);
            __syncwarp();
        }
    }
    if ((ja ^ jb) == 0xFFFFFFFFu) sink[0] = ja;
}

int main(int argc, char **argv) {
    cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
    const uint32_t N = argc > 1 ? (uint32_t)atoi(argv[1]) : 8192;
    const uint32_t slots = argc > 2 ? (uint32_t)atoi(argv[2]) : (uint32_t)p.multiProcessorCount * TPB;
    const int pairs = argc > 3 ? atoi(argv[3]) : 3;
    if (N < 2 || (N & (N - 1)) || slots == 0 || slots % 32) { printf("{\"error\": \"N must be a power of two >= 2, slots a multiple of 32\"}\n"); return 1; }
    const size_t bytes = (size_t)slots * 2 * 128 * N;   // two N-row scratchpads per slot
    uint4 *V; uint32_t *sink;
    CK(cudaMalloc(&V, bytes));
    CK(cudaMalloc(&sink, 4));
    CK(cudaMemset(V, 0, bytes));
    const size_t smem = TPB / 32 * 8192;
    CK(cudaFuncSetAttribute(traffic<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaFuncSetAttribute(traffic<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const uint32_t grid = (slots + TPB - 1) / TPB;
    cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    auto run = [&](bool phased) {
        CK(cudaEventRecord(a));
        if (phased) traffic<true><<<grid, TPB, smem>>>(V, N, slots, sink);
        else traffic<false><<<grid, TPB, smem>>>(V, N, slots, sink);
        CK(cudaGetLastError());
        CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
        float ms; CK(cudaEventElapsedTime(&ms, a, b));
        const double moved = (double)slots * (phased ? 2 : 1) * 2 * 128 * N;
        return std::make_pair(ms, moved / (ms * 1e-3) / 1e9);
    };
    run(false); run(true);   // warm-up: module load, first touch of every page
    printf("{\"device\": \"%s\", \"sms\": %d, \"N\": %u, \"slots\": %u, \"tpb\": %d, \"scratch_gib\": %.2f}\n", p.name,
           p.multiProcessorCount, N, slots, TPB, bytes / 1073741824.0);
    for (int r = 0; r < pairs; r++)
        for (int phased = 0; phased < 2; phased++) {
            const auto m = run(phased != 0);
            printf("{\"schedule\": \"%s\", \"rep\": %d, \"ms\": %.3f, \"GB_per_s\": %.1f}\n", phased ? "phased" : "interleaved", r,
                   m.first, m.second);
        }
    return 0;
}
