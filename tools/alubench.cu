// tools/alubench.cu — dev probe: issue rate of the instruction classes Salsa20/8 is made of on this GPU.
//   mode 0: SHF.L.W (rotate) only      mode 1: LOP3 (xor) only      mode 2: IMAD.IADD-style add only
//   mode 3: the Salsa mix — add, rotate, xor per step (8 independent chains per thread)
// Prints thread-instructions per clock per SM; the alu pipe (SHF, LOP3) tops out at 64, which is the ceiling
// the ROMix kernel runs into (DESIGN.md §4).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/alubench tools/alubench.cu
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

template <int MODE>
__global__ void __launch_bounds__(256) probe(uint32_t *out, int iters, uint32_t seed) {
    uint32_t x[8], y[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { x[i] = seed + threadIdx.x * 8 + i; y[i] = seed * 3 + i + blockIdx.x; }
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int r = 0; r < 16; r++) {
#pragma unroll
            for (int i = 0; i < 8; i++) {
                // asm volatile: every op must survive as one SASS instruction (no folding of rotate chains)
                if (MODE == 0) asm volatile("shf.l.wrap.b32 %0, %0, %0, 7;" : "+r"(x[i]));
                else if (MODE == 1) asm volatile("lop3.b32 %0, %0, %1, %2, 0xE8;" : "+r"(x[i]) : "r"(y[i]), "r"(y[(i + 3) & 7]));   // majority: not foldable
                else if (MODE == 2) asm volatile("add.u32 %0, %0, %1;" : "+r"(x[i]) : "r"(y[i]));
                else {
                    uint32_t s;
                    asm volatile("add.u32 %0, %1, %2;" : "=r"(s) : "r"(x[i]), "r"(y[(i + 1) & 7]));
                    asm volatile("shf.l.wrap.b32 %0, %0, %0, 7;" : "+r"(s));
                    asm volatile("xor.b32 %0, %0, %1;" : "+r"(y[i]) : "r"(s));
                }
            }
        }
    }
    uint32_t a = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) a ^= x[i] ^ y[i];
    if (a == 0x12345678) out[0] = a;
}

template <int MODE>
static void run(const char *name, double instr_per_inner, int sms, double ghz) {
    uint32_t *d; cudaMalloc(&d, 4);
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    const int iters = 4000, grid = sms * 8;
    probe<MODE><<<grid, 256>>>(d, 100, 1);
    cudaEventRecord(a);
    probe<MODE><<<grid, 256>>>(d, iters, 2);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    const double instr = (double)grid * 256 * iters * 16 * 8 * instr_per_inner;
    printf("%-28s %8.1f G thread-instr/s  = %6.1f per clk per SM at %.2f GHz\n", name, instr / ms / 1e6, instr / ms / 1e6 / sms / ghz, ghz);
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    const double ghz = khz / 1e6;
    printf("%s, %d SMs, nominal %.3f GHz (rates per clock use the nominal clock)\n", p.name, p.multiProcessorCount, ghz);
    run<0>("SHF rotate only", 1, p.multiProcessorCount, ghz);
    run<1>("LOP3 only", 1, p.multiProcessorCount, ghz);
    run<2>("integer add only", 1, p.multiProcessorCount, ghz);
    run<3>("salsa step add+rot+xor", 3, p.multiProcessorCount, ghz);
    return 0;
}
