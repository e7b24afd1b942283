// gsb_scene.cu -- scene ingest: GSScene::Vertex AoS -> device layouts + cov3D precompute.
// Replaces vertexBuffer->uploadFrom (src/GSScene.cpp:61) and the precomp_cov3d dispatch
// (src/GSScene.cpp:157-184, src/shaders/precomp_cov3d.comp:25-48, common.glsl:51-75).
// Load-time only (once per scene).  Compiled with -fmad=false: every op is one IEEE operation
// so the result equals the oracle's generic mat3 products (zero terms dropped: x + 0 == x).
#include <cuda_fp16.h>

#include "gsb_geom.cuh"
#include "gsb_internal.cuh"

namespace gsb {

template <bool SH16>
__global__ void __launch_bounds__(256) k_ingest_cov3d(const float4* __restrict__ vtx, uint64_t count,
                                                      uint64_t dst_offset, float4* __restrict__ pos_op,
                                                      float4* __restrict__ cov_a, float2* __restrict__ cov_b,
                                                      float4* __restrict__ sh, float scale_factor) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const float4* v = vtx + i * 15;  // 60 floats = 15 float4
    const float4 p = v[0];           // position (xyz, 1)
    const float4 so = v[1];          // scale_opacity
    const float4 q = v[2];           // rotation: x = w (common.glsl:52-55)
    const uint64_t o = dst_offset + i;
    store_cov3d(p, so, q, o, pos_op, cov_a, cov_b, scale_factor);
    if constexpr (SH16) {  // gsb_set_sh_storage(1): 48 halves = 6 x 16 B per Gaussian (non-parity)
        uint4* dsh = reinterpret_cast<uint4*>(sh) + o * 6;
#pragma unroll
        for (int k = 0; k < 6; k++) {
            const float4 a = v[3 + 2 * k], b = v[4 + 2 * k];
            const __half2 h0 = __floats2half2_rn(a.x, a.y), h1 = __floats2half2_rn(a.z, a.w), h2 = __floats2half2_rn(b.x, b.y),
                          h3 = __floats2half2_rn(b.z, b.w);
            dsh[k] = make_uint4(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1),
                                *reinterpret_cast<const uint32_t*>(&h2), *reinterpret_cast<const uint32_t*>(&h3));
        }
    } else {
        float4* dsh = sh + o * 12;
#pragma unroll
        for (int k = 0; k < 12; k++) dsh[k] = v[3 + k];
    }
}

cudaError_t launch_cov3d(const float* vtx_aos, uint64_t count, uint64_t dst_offset, float4* pos_op,
                         float4* cov_a, float2* cov_b, float* sh, float scale_factor, cudaStream_t s, bool sh_half) {
    if (count == 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((count + 255) / 256);
    if (sh_half)
        k_ingest_cov3d<true><<<blocks, 256, 0, s>>>(reinterpret_cast<const float4*>(vtx_aos), count, dst_offset, pos_op, cov_a, cov_b,
                                                    reinterpret_cast<float4*>(sh), scale_factor);
    else
        k_ingest_cov3d<false><<<blocks, 256, 0, s>>>(reinterpret_cast<const float4*>(vtx_aos), count, dst_offset, pos_op, cov_a, cov_b,
                                                     reinterpret_cast<float4*>(sh), scale_factor);
    return cudaGetLastError();
}

}  // namespace gsb
