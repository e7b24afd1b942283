// Microbenchmark: throughput of the building blocks a radix-rank can be made of, per SM, on sm_90a:
//   ATOMS.OR / ATOMS.ADD to spread shared-memory addresses (one per lane), plain LDS / STS, __match_any_sync,
//   and the 8-ballot digit match.  Prints cycles per warp-instruction per SM with 8 and 16 resident warps.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o smem_atomic smem_atomic.cu
#include <cstdio>
#include <cuda_runtime.h>
constexpr int ITERS = 2048;
template <int MODE>
__global__ void k(unsigned* out, long long* cyc, unsigned seed) {
    __shared__ unsigned s[8192];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < 8192; i += blockDim.x) s[i] = 0;
    __syncthreads();
    unsigned x = seed * 2654435761u + tid * 40503u, acc = 0;
    const long long t0 = clock64();
#pragma unroll 4
    for (int it = 0; it < ITERS; it++) {
        x = x * 1664525u + 1013904223u;
        const unsigned d = (x >> 13) & 255u;                    // pseudo-random 8-bit digit
        unsigned* p = &s[warp * 256 + d];                        // per-warp region, like the sort's match / counter arrays
        if (MODE == 0) atomicOr(p, 1u << lane);
        if (MODE == 1) acc += atomicAdd(p, 1u);
        if (MODE == 2) acc += *(volatile unsigned*)p;
        if (MODE == 3) *(volatile unsigned*)p = x;
        if (MODE == 4) acc += __match_any_sync(0xffffffffu, d);
        if (MODE == 5) {
            unsigned m = 0xffffffffu;
#pragma unroll
            for (int b = 0; b < 8; b++) {
                const bool bit = (d >> b) & 1u;
                const unsigned v = __ballot_sync(0xffffffffu, bit);
                m &= bit ? v : ~v;
            }
            acc += m;
        }
        if (MODE == 6) {  // distinct banks: lane-private address (no conflicts at all)
            atomicOr(&s[warp * 256 + ((lane + it) & 31) + (d & 0xe0u)], 1u << lane);
        }
        if (MODE == 7) {  // atomicOr + read back + clear, the sort's sequence
            atomicOr(p, 1u << lane);
            __syncwarp();
            const unsigned peers = *(volatile unsigned*)p;
            __syncwarp();
            if (lane == __ffs(peers) - 1) *(volatile unsigned*)p = 0u;
            acc += peers;
            __syncwarp();
        }
    }
    const long long t1 = clock64();
    if (tid == 0) cyc[blockIdx.x] = t1 - t0;
    out[blockIdx.x * blockDim.x + tid] = acc + s[tid];
}
template <int MODE>
void run(const char* name) {
    unsigned* out; long long* cyc;
    cudaMalloc(&out, 132 * 2 * 512 * 4); cudaMalloc(&cyc, 132 * 2 * 8);
    for (int threads : {256, 512}) for (int ctas : {1, 2}) {
        k<MODE><<<132 * ctas, threads>>>(out, cyc, 1); cudaDeviceSynchronize();
        k<MODE><<<132 * ctas, threads>>>(out, cyc, 2); cudaDeviceSynchronize();
        long long h[264]; cudaMemcpy(h, cyc, 132 * ctas * 8, cudaMemcpyDeviceToHost);
        double avg = 0; for (int i = 0; i < 132 * ctas; i++) avg += h[i]; avg /= 132 * ctas;
        const double warp_instr_per_sm = (double)ITERS * (threads / 32) * ctas;
        printf("%-34s threads %3d x %d CTA/SM: %7.2f cycles per warp-op per SM (%.2f per lane)\n", name, threads, ctas, avg / warp_instr_per_sm, avg / warp_instr_per_sm / 32);
    }
    cudaFree(out); cudaFree(cyc);
}
int main() {
    run<0>("ATOMS.OR random digit (per warp)");
    run<6>("ATOMS.OR conflict-free banks");
    run<1>("ATOMS.ADD+return random digit");
    run<2>("LDS random digit");
    run<3>("STS random digit");
    run<4>("match.any 8-bit digit");
    run<5>("8-ballot match");
    run<7>("atomicOr+readback+clear sequence");
    return 0;
}
