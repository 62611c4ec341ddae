// bench_tex_gather.cu — A/B for the 2x2 bilinear gather of the warp kernel's 8-bit sampler (north_star: "tex2D only where it wins on ncu";
// VERDICT r1 asks for one recorded comparison).  Same exact integer blend (5-bit weights, sample_u8_bilinear in warp_kernel.cuh) fed by
//   A) four read-only LDG.32 taps (what the kernel does)            B) four tex2D<uchar4> POINT fetches from a pitch-2D texture object
//   C) four tex2Dgather<uchar4> (one per channel: the four taps of that channel in one fetch)
// over a 3840x2160 RGBA8 frame with a warp-like coordinate field (smooth, ~1 degree of roll + barrel curvature, 1/32-pixel steps).
// Hardware bilinear filtering is not an option: its 8-bit weights and internal rounding are not the reference's arithmetic.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo tools/bench_tex_gather.cu -o /tmp/bench_tex_gather ; run on the GPU.
// Static instruction counts: cuobjdump -sass /tmp/bench_tex_gather | grep -c ... (recorded in DESIGN.md §4).
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cstdint>

#define W 3840
#define H 2160

__device__ __forceinline__ void coords(int x, int y, int& sx0, int& sy0) {
    // source position in 1/32 px: identity + roll + a barrel term; stays inside [1, W - 2] x [1, H - 2]
    const float fx = (float)x - 1920.0f, fy = (float)y - 1080.0f;
    const float r2 = (fx * fx + fy * fy) * (1.0f / (1920.0f * 1920.0f));
    const float s = 0.96f - 0.03f * r2;
    const float u = 1920.0f + s * (fx * 0.99985f - fy * 0.01745f), v = 1080.0f + s * (fx * 0.01745f + fy * 0.99985f);
    sx0 = min(max(__float2int_rn(u * 32.0f), 32), (W - 2) * 32); sy0 = min(max(__float2int_rn(v * 32.0f), 32), (H - 2) * 32);
}
__device__ __forceinline__ uint32_t blend(uint32_t p00, uint32_t p01, uint32_t p10, uint32_t p11, int sx0, int sy0) {
    const uint32_t fx = (uint32_t)sx0 & 31u, fy = (uint32_t)sy0 & 31u, wx0 = 32u - fx, wx1 = fx, wy = (32u - fy) | (fy << 8);
    const uint32_t he0 = (p00 & 0x00ff00ffu) * wx0 + (p01 & 0x00ff00ffu) * wx1, he1 = (p10 & 0x00ff00ffu) * wx0 + (p11 & 0x00ff00ffu) * wx1;
    const uint32_t ho0 = __byte_perm(p00, 0u, 0x4341) * wx0 + __byte_perm(p01, 0u, 0x4341) * wx1, ho1 = __byte_perm(p10, 0u, 0x4341) * wx0 + __byte_perm(p11, 0u, 0x4341) * wx1;
    const uint32_t n0 = __dp2a_lo(__byte_perm(he0, he1, 0x5410), wy, 0u) >> 10, n2 = __dp2a_lo(__byte_perm(he0, he1, 0x7632), wy, 0u) >> 10;
    const uint32_t n1 = __dp2a_lo(__byte_perm(ho0, ho1, 0x5410), wy, 0u) >> 10, n3 = __dp2a_lo(__byte_perm(ho0, ho1, 0x7632), wy, 0u) >> 10;
    return n0 | (n1 << 8) | (n2 << 16) | (n3 << 24);
}
__global__ void __launch_bounds__(128) k_ldg(const uint8_t* __restrict__ src, int stride, uint32_t* __restrict__ dst) {
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 4 + threadIdx.y;
    int sx0, sy0; coords(x, y, sx0, sy0);
    const uint8_t* r0 = src + (long long)(sy0 >> 5) * stride + (long long)(sx0 >> 5) * 4; const uint8_t* r1 = r0 + stride;
    const uint32_t p00 = __ldg((const uint32_t*)r0), p01 = __ldg((const uint32_t*)(r0 + 4)), p10 = __ldg((const uint32_t*)r1), p11 = __ldg((const uint32_t*)(r1 + 4));
    dst[(size_t)y * W + x] = blend(p00, p01, p10, p11, sx0, sy0);
}
__device__ __forceinline__ uint32_t pk(uchar4 c) { return (uint32_t)c.x | ((uint32_t)c.y << 8) | ((uint32_t)c.z << 16) | ((uint32_t)c.w << 24); }
__global__ void __launch_bounds__(128) k_tex(cudaTextureObject_t tex, uint32_t* __restrict__ dst) {
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 4 + threadIdx.y;
    int sx0, sy0; coords(x, y, sx0, sy0);
    const float tx = (float)(sx0 >> 5), ty = (float)(sy0 >> 5);
    const uint32_t p00 = pk(tex2D<uchar4>(tex, tx, ty)), p01 = pk(tex2D<uchar4>(tex, tx + 1.0f, ty));
    const uint32_t p10 = pk(tex2D<uchar4>(tex, tx, ty + 1.0f)), p11 = pk(tex2D<uchar4>(tex, tx + 1.0f, ty + 1.0f));
    dst[(size_t)y * W + x] = blend(p00, p01, p10, p11, sx0, sy0);
}
__global__ void __launch_bounds__(128) k_gather(cudaTextureObject_t tex, uint32_t* __restrict__ dst) {
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 4 + threadIdx.y;
    int sx0, sy0; coords(x, y, sx0, sy0);
    // gather returns (x0,y1), (x1,y1), (x1,y0), (x0,y0) of one channel around the texel corner at (tx + 1, ty + 1)
    const float tx = (float)(sx0 >> 5) + 1.0f, ty = (float)(sy0 >> 5) + 1.0f;
    const uchar4 g0 = tex2Dgather<uchar4>(tex, tx, ty, 0), g1 = tex2Dgather<uchar4>(tex, tx, ty, 1), g2 = tex2Dgather<uchar4>(tex, tx, ty, 2), g3 = tex2Dgather<uchar4>(tex, tx, ty, 3);
    const uint32_t p00 = (uint32_t)g0.w | ((uint32_t)g1.w << 8) | ((uint32_t)g2.w << 16) | ((uint32_t)g3.w << 24);
    const uint32_t p01 = (uint32_t)g0.z | ((uint32_t)g1.z << 8) | ((uint32_t)g2.z << 16) | ((uint32_t)g3.z << 24);
    const uint32_t p10 = (uint32_t)g0.x | ((uint32_t)g1.x << 8) | ((uint32_t)g2.x << 16) | ((uint32_t)g3.x << 24);
    const uint32_t p11 = (uint32_t)g0.y | ((uint32_t)g1.y << 8) | ((uint32_t)g2.y << 16) | ((uint32_t)g3.y << 24);
    dst[(size_t)y * W + x] = blend(p00, p01, p10, p11, sx0, sy0);
}

int main() {
    const int stride = W * 4, ring = 8;
    std::vector<uint8_t*> src(ring); std::vector<cudaTextureObject_t> tex(ring);
    std::vector<uint8_t> h((size_t)stride * H);
    for (int r = 0; r < ring; ++r) {
        uint32_t s = 12345u + r;
        for (auto& b : h) { s = s * 1664525u + 1013904223u; b = (uint8_t)(s >> 24); }
        cudaMalloc(&src[r], h.size()); cudaMemcpy(src[r], h.data(), h.size(), cudaMemcpyHostToDevice);
        cudaResourceDesc rd = {}; rd.resType = cudaResourceTypePitch2D; rd.res.pitch2D.devPtr = src[r]; rd.res.pitch2D.desc = cudaCreateChannelDesc<uchar4>();
        rd.res.pitch2D.width = W; rd.res.pitch2D.height = H; rd.res.pitch2D.pitchInBytes = stride;
        cudaTextureDesc td = {}; td.addressMode[0] = td.addressMode[1] = cudaAddressModeClamp; td.filterMode = cudaFilterModePoint; td.readMode = cudaReadModeElementType; td.normalizedCoords = 0;
        if (cudaCreateTextureObject(&tex[r], &rd, &td, nullptr) != cudaSuccess) { printf("texture object failed: %s\n", cudaGetErrorString(cudaGetLastError())); return 1; }
    }
    uint32_t *d0, *d1, *d2; cudaMalloc(&d0, (size_t)W * H * 4); cudaMalloc(&d1, (size_t)W * H * 4); cudaMalloc(&d2, (size_t)W * H * 4);
    const dim3 block(32, 4), grid(W / 32, H / 4);
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    float ms[3] = {0, 0, 0};
    for (int variant = 0; variant < 3; ++variant) {
        for (int rep = 0; rep < 2; ++rep) {
            cudaEventRecord(a);
            for (int i = 0; i < 200; ++i) {
                if (variant == 0) k_ldg<<<grid, block>>>(src[i % ring], stride, d0);
                else if (variant == 1) k_tex<<<grid, block>>>(tex[i % ring], d1);
                else k_gather<<<grid, block>>>(tex[i % ring], d2);
            }
            cudaEventRecord(b); cudaEventSynchronize(b);
            cudaEventElapsedTime(&ms[variant], a, b);
        }
    }
    std::vector<uint32_t> o0((size_t)W * H), o1((size_t)W * H), o2((size_t)W * H);
    k_ldg<<<grid, block>>>(src[0], stride, d0); k_tex<<<grid, block>>>(tex[0], d1); k_gather<<<grid, block>>>(tex[0], d2);
    cudaMemcpy(o0.data(), d0, o0.size() * 4, cudaMemcpyDeviceToHost); cudaMemcpy(o1.data(), d1, o1.size() * 4, cudaMemcpyDeviceToHost); cudaMemcpy(o2.data(), d2, o2.size() * 4, cudaMemcpyDeviceToHost);
    size_t bad1 = 0, bad2 = 0; for (size_t i = 0; i < o0.size(); ++i) { bad1 += o0[i] != o1[i]; bad2 += o0[i] != o2[i]; }
    printf("{\"ldg_us_per_frame\": %.2f, \"tex2d_point_us_per_frame\": %.2f, \"tex2dgather_us_per_frame\": %.2f, \"tex_mismatches\": %zu, \"gather_mismatches\": %zu, \"error\": \"%s\"}\n",
           ms[0] * 5.0f, ms[1] * 5.0f, ms[2] * 5.0f, bad1, bad2, cudaGetErrorString(cudaGetLastError()));
    return 0;
}
