// smem_atomics_microbench.cu — how expensive is RED.SHARED.ADD (ATOMS / ATOMS.POPC.INC) per warp instruction as a
// function of the lanes' address pattern?  Input for the counting design of kta::scan_kernel (DESIGN.md §5.1):
// per-lane bucket increments hit few distinct addresses when a tile lies inside one partition run, and many
// addresses in few banks when P is large.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/smem_atomics tools/smem_atomics_microbench.cu && build/smem_atomics   (after mkdir -p build)
//
// Prints, per pattern, cycles per warp-level atomic instruction with 32 resident warps per SM (like the scan kernel)
// and with 1 warp (latency view).  Patterns: the address each lane uses, in 4-byte words.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

enum Pattern {
    ALL_SAME,          // 32 lanes, one address                      (one partition, one size bucket)
    TWO_ADDR,          // two addresses, 16 lanes each                (one partition, two size buckets)
    FOUR_ADDR,         // four addresses in four banks
    DISTINCT_BANKS,    // 32 addresses, 32 banks                      (conflict-free scatter)
    SAME_BANK_2,       // 32 addresses, 16 banks (2-way conflict)
    SAME_BANK_8,       // 32 addresses, 4 banks (8-way conflict)      (P = 256: eight columns per bank)
    SAME_BANK_32,      // 32 addresses, one bank (32-way conflict)
    RANDOM_64,         // random column of 64 (P = 64), fixed row
    RANDOM_256,        // random column of 256 (P = 256), fixed row
    N_PATTERNS
};
static const char *NAMES[N_PATTERNS] = {"all lanes one address", "two addresses", "four addresses", "32 addresses / 32 banks",
                                        "32 addresses / 16 banks", "32 addresses / 4 banks", "32 addresses / 1 bank",
                                        "random of 64 columns", "random of 256 columns"};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void red_add(uint32_t a, uint32_t v) { asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

template <bool INC_ONE>
__global__ void __launch_bounds__(1024, 1) bench(int pattern, int iters, unsigned long long *cycles, uint32_t *sink) {
    extern __shared__ uint32_t s[];
    for (int i = threadIdx.x; i < 8192; i += blockDim.x) s[i] = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t rnd = (threadIdx.x + 1) * 2654435761u + blockIdx.x * 40503u;
    uint32_t w;
    switch (pattern) {
        case ALL_SAME: w = 7; break;
        case TWO_ADDR: w = 7 + (lane >> 4); break;
        case FOUR_ADDR: w = 7 + (lane >> 3); break;
        case DISTINCT_BANKS: w = lane; break;
        case SAME_BANK_2: w = (lane & 15) + 32 * (lane >> 4); break;
        case SAME_BANK_8: w = (lane & 3) + 32 * (lane >> 2); break;
        case SAME_BANK_32: w = 32 * lane; break;
        default: w = 0; break;
    }
    const uint32_t base = smem_u32(s) + 4u * (uint32_t)(warp & 3) * 2048u;   // four row groups, like different counter rows
    const unsigned long long t0 = clock64();
    for (int i = 0; i < iters; i++) {
        if (pattern >= RANDOM_64) {
            rnd = rnd * 1664525u + 1013904223u;
            w = (rnd >> 16) % (pattern == RANDOM_64 ? 64u : 256u);
        }
        red_add(base + 4u * w, INC_ONE ? 1u : (rnd | 1u));
    }
    __syncthreads();
    const unsigned long long t1 = clock64();
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
    if (threadIdx.x < 64) sink[blockIdx.x * 64 + threadIdx.x] = s[threadIdx.x];
}

int main() {
    int dev = 0, sms = 0;
    CK(cudaSetDevice(dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    unsigned long long *d_cycles;
    uint32_t *d_sink;
    CK(cudaMalloc(&d_cycles, sms * sizeof(unsigned long long)));
    CK(cudaMalloc(&d_sink, sms * 64 * 4));
    const int iters = 20000;
    printf("%-28s %22s %22s %22s\n", "pattern", "cyc/instr 32 warps +1", "cyc/instr 32 warps +v", "cyc/instr 1 warp +1");
    for (int p = 0; p < N_PATTERNS; p++) {
        double r[3];
        for (int variant = 0; variant < 3; variant++) {
            const int threads = variant == 2 ? 32 : 1024;
            for (int rep = 0; rep < 2; rep++) {   // first repetition warms up
                if (variant == 1) bench<false><<<sms, threads, 32768>>>(p, iters, d_cycles, d_sink);
                else bench<true><<<sms, threads, 32768>>>(p, iters, d_cycles, d_sink);
                CK(cudaDeviceSynchronize());
            }
            unsigned long long c = 0;
            CK(cudaMemcpy(&c, d_cycles, 8, cudaMemcpyDeviceToHost));
            r[variant] = (double)c / ((double)iters * (threads / 32));
        }
        printf("%-28s %22.2f %22.2f %22.2f\n", NAMES[p], r[0], r[1], r[2]);
    }
    return 0;
}
