// tools/membench.cu — dev probe: what HBM delivers for the two ROMix access patterns on this GPU.
//   (a) random 128-byte row reads (one row per 8-lane group, 16 B per lane) over a large buffer,
//       with `depth` independent rows in flight per group;
//   (b) streaming 128-bit writes; (c) both at once (half the CTAs each).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/membench tools/membench.cu
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>

__device__ __forceinline__ uint4 ld_cs(const uint4 *p) {
    uint4 v; asm volatile("ld.global.cs.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p)); return v;
}
__device__ __forceinline__ void st_cs(uint4 *p, uint4 v) {
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// mode bit0: readers, bit1: writers.  rows = number of 128-B rows in the buffer (power of two).
template <int DEPTH>
__global__ void __launch_bounds__(128) probe(uint4 *buf, uint64_t rows, int iters, int mode, uint32_t *sink, int dependent) {
    const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t grp = gid >> 3, c = gid & 7;
    const bool writer = (mode == 2) || (mode == 3 && (blockIdx.x & 1));
    uint32_t acc = 0;
    if (!writer) {
        uint64_t s[DEPTH];
#pragma unroll
        for (int d = 0; d < DEPTH; d++) s[d] = (uint64_t)grp * 0x9E3779B97F4A7C15ull + d * 0xD1B54A32D192ED03ull + 12345;
        for (int it = 0; it < iters; it++) {
            uint4 v[DEPTH];
#pragma unroll
            for (int d = 0; d < DEPTH; d++) {
                s[d] = s[d] * 6364136223846793005ull + 1442695040888963407ull;
                const uint64_t row = (s[d] >> 20) & (rows - 1);
                v[d] = ld_cs(buf + row * 8 + c);
            }
#pragma unroll
            for (int d = 0; d < DEPTH; d++) {
                acc += v[d].x ^ v[d].y ^ v[d].z ^ v[d].w;
                if (dependent) s[d] ^= (uint64_t)(__shfl_sync(0xffffffffu, v[d].x, threadIdx.x & 24) & 0xff) << 40;   // next address depends on the data
            }
        }
    } else {
        // each warp streams 512 contiguous bytes per store instruction over its own region
        const uint64_t warp = gid >> 5, lane = gid & 31;
        const uint64_t warps = (uint64_t)gridDim.x * blockDim.x / 32;
        const uint64_t per = rows * 8 / warps;   // uint4 per warp
        uint4 *base = buf + warp * per;
        for (int it = 0; it < iters * DEPTH; it++) {
            const uint64_t off = ((uint64_t)it * 32) % (per - 32);
            st_cs(base + off + lane, make_uint4(it, gid, 3, 4));
        }
    }
    if (acc == 0xdeadbeef) sink[0] = acc;
}

int main(int argc, char **argv) {
    const double gib = argc > 1 ? atof(argv[1]) : 64.0;
    uint64_t rows = 1; while ((rows * 2) * 128 <= (uint64_t)(gib * (1ull << 30))) rows *= 2;
    uint4 *buf; uint32_t *sink;
    if (cudaMalloc(&buf, rows * 128) != cudaSuccess) { printf("alloc failed\n"); return 1; }
    cudaMalloc(&sink, 4);
    cudaMemset(buf, 1, rows * 128);
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    printf("buffer %.1f GiB (%llu rows)\n", rows * 128 / 1073741824.0, (unsigned long long)rows);
    for (int mode = 1; mode <= 3; mode++)
        for (int dep = 0; dep <= (mode == 2 ? 0 : 1); dep++)
            for (int ctas = 2; ctas <= 8; ctas += 2) {
                const int grid = p.multiProcessorCount * ctas, iters = 2000;
                probe<1><<<grid, 128>>>(buf, rows, 50, mode, sink, dep);
                cudaEventRecord(a);
                probe<1><<<grid, 128>>>(buf, rows, iters, mode, sink, dep);
                cudaEventRecord(b); cudaEventSynchronize(b);
                float ms; cudaEventElapsedTime(&ms, a, b);
                const double bytes = (double)grid * 128 * iters * 16;
                printf("mode %d (%s) dependent=%d ctas/SM=%d depth=1: %.0f GB/s\n", mode, mode == 1 ? "random 128B reads" : mode == 2 ? "streaming writes" : "half/half", dep, ctas, bytes / ms / 1e6);
                if (mode != 2) {
                    probe<4><<<grid, 128>>>(buf, rows, iters / 4, mode, sink, dep);
                    cudaEventRecord(a);
                    probe<4><<<grid, 128>>>(buf, rows, iters / 4, mode, sink, dep);
                    cudaEventRecord(b); cudaEventSynchronize(b);
                    cudaEventElapsedTime(&ms, a, b);
                    printf("mode %d dependent=%d ctas/SM=%d depth=4: %.0f GB/s\n", mode, dep, ctas, bytes / ms / 1e6);
                }
            }
    return 0;
}
