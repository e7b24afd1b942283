// Reference point for the instance sort (NOT product code; CUB is library code and never on the frame path):
// cub::DeviceRadixSort::SortPairs (Onesweep in CUDA 12.9) vs libgsb200's gsb_sort_pairs32 on the frame's shapes:
//   (a) M = 17.2 M pairs, 15 key bits (tile ids of 3200x1400), keys skewed like a tile histogram,
//   (b) N_v = 2.56 M pairs, 32 key bits (depth bits).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -I../../include -o cub_sort cub_sort.cu -L../../3dgs.cpp_b200 -lgsb200 -Xlinker -rpath,'$ORIGIN/../../3dgs.cpp_b200'
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cub/device/device_radix_sort.cuh>
#include "gs_b200.h"

static uint64_t s = 88172645463325252ull;
static uint32_t rnd() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return (uint32_t)(s >> 11); }

static void run(gsb_ctx* ctx, size_t m, int bits, bool depth_like) {
    std::vector<uint32_t> hk(m), hv(m);
    for (size_t i = 0; i < m; i++) {
        if (depth_like) { float d = 4.0f + 20.0f * (rnd() / 2097152.0f / 1024.0f); memcpy(&hk[i], &d, 4); }
        else hk[i] = rnd() % 17600u;
        hv[i] = (uint32_t)i;
    }
    uint32_t *k0, *k1, *v0, *v1, *ki, *vi;
    cudaMalloc(&k0, m * 4); cudaMalloc(&k1, m * 4); cudaMalloc(&v0, m * 4); cudaMalloc(&v1, m * 4); cudaMalloc(&ki, m * 4); cudaMalloc(&vi, m * 4);
    cudaMemcpy(ki, hk.data(), m * 4, cudaMemcpyHostToDevice); cudaMemcpy(vi, hv.data(), m * 4, cudaMemcpyHostToDevice);
    size_t tmp_bytes = 0;
    cub::DoubleBuffer<uint32_t> dk(k0, k1), dv(v0, v1);
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, dk, dv, (int)m, 0, bits);
    void* tmp; cudaMalloc(&tmp, tmp_bytes);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float best_cub = 1e9f, best_gsb = 1e9f;
    for (int it = 0; it < 12; it++) {
        cudaMemcpy(k0, ki, m * 4, cudaMemcpyDeviceToDevice); cudaMemcpy(v0, vi, m * 4, cudaMemcpyDeviceToDevice);
        cub::DoubleBuffer<uint32_t> a(k0, k1), b(v0, v1);
        cudaDeviceSynchronize();
        cudaEventRecord(e0);
        cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, a, b, (int)m, 0, bits);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (it >= 2 && ms < best_cub) best_cub = ms;
    }
    cudaStream_t st; cudaStreamCreate(&st);
    for (int it = 0; it < 12; it++) {
        cudaMemcpy(k0, ki, m * 4, cudaMemcpyDeviceToDevice); cudaMemcpy(v0, vi, m * 4, cudaMemcpyDeviceToDevice);
        cudaDeviceSynchronize();
        cudaEventRecord(e0, st);
        int rc = gsb_sort_pairs32(ctx, k0, v0, k1, v1, m, bits, st);  // includes its own status alloc + memset + final sync
        cudaEventRecord(e1, st); cudaEventSynchronize(e1);
        if (rc) { printf("gsb_sort_pairs32 rc %d %s\n", rc, gsb_last_error(ctx)); break; }
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (it >= 2 && ms < best_gsb) best_gsb = ms;
    }
    const double bytes = (double)m * (4 + 16.0 * ((bits + 7) / 8));
    printf("m=%zu bits=%d %s: cub %.4f ms (%.0f GB/s alg)  gsb_sort_pairs32 %.4f ms (%.0f GB/s alg; includes alloc/memset/sync of the standalone entry point)\n",
           m, bits, depth_like ? "depth-like" : "tile-like", best_cub, bytes / best_cub / 1e6, best_gsb, bytes / best_gsb / 1e6);
    cudaFree(k0); cudaFree(k1); cudaFree(v0); cudaFree(v1); cudaFree(ki); cudaFree(vi); cudaFree(tmp);
}

int main() {
    gsb_ctx* ctx = nullptr;
    if (gsb_create(0, &ctx)) { printf("no device\n"); return 1; }
    run(ctx, 17229065, 15, false);
    run(ctx, 17229065, 16, false);
    run(ctx, 2558286, 32, true);
    run(ctx, 30364152, 15, false);
    gsb_destroy(ctx);
    return 0;
}
