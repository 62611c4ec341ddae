// selftest.cu — device-side check of the packed f32x2 primitives against the scalar operations they replace.
// gf_cuda_selftest(device, n, out[4]): n pseudo-random operand pairs per primitive; out = mismatch counts for
// {div_exact_checked vs '/', sqrt_exact vs sqrtf, atanf2 vs gf_atanf, div_uniform vs '/'}.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <algorithm>
#include <vector>
#include "../../include/gyroflow_cuda.h"
#include "warp_kernel_x2.cuh"
#include "sync_select.cuh"
#include "c_abi_internal.h"

using namespace gf;

namespace {
inline uint32_t __float_as_uint_host(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
__device__ __forceinline__ uint32_t mix(uint64_t v) {
    v ^= v >> 33; v *= 0xff51afd7ed558ccdULL; v ^= v >> 33; v *= 0xc4ceb9fe1a85ec53ULL; v ^= v >> 33;
    return (uint32_t)v;
}
// operand generator: a mix of fully random bit patterns, "coordinate-like" magnitudes and values near 1
__device__ __forceinline__ float gen(uint64_t i, uint32_t salt) {
    const uint32_t h = mix(i * 0x9E3779B97F4A7C15ULL + salt);
    const uint32_t sel = mix(i + 77u * salt) & 7u;
    if (sel < 3) return __uint_as_float(h);                                             // anything, incl. NaN/inf/denormals
    if (sel < 6) return __uint_as_float((h & 0x807fffffu) | ((100u + (mix(i ^ salt) % 56u)) << 23));   // 2^-27 .. 2^28
    return __uint_as_float((h & 0x007fffffu) | 0x3f800000u) - ((h >> 31) ? 0.0f : 1.0f);        // [1,2) or [0,1)
}
__device__ __forceinline__ bool same(float a, float b) { return __float_as_uint(a) == __float_as_uint(b) || (a != a && b != b); }

__global__ void selftest_kernel(unsigned long long n, unsigned long long seed, unsigned long long* out, uint32_t* dbg) {
    __shared__ p2::AtanRow tab[p2::ATAN_ROWS];
    p2::atan_table_init(tab, threadIdx.x, blockDim.x);
    __syncthreads();
    unsigned long long bad[4] = {0, 0, 0, 0};
    if (blockIdx.x == 0 && threadIdx.x < p2::ATAN_ROWS) {       // the literal table in global memory == the computed rows
        const p2::AtanRow& g = p2::GF_ATAN_TAB[threadIdx.x]; const p2::AtanRow& c = tab[threadIdx.x];
        if (!(same(g.A, c.A) && same(g.B, c.B) && same(g.C, c.C) && same(g.D, c.D) && same(g.hi, c.hi) && same(g.lo, c.lo))) bad[2]++;
    }
    MapC m; m.in_min = 0.0f; m.mul = 1.0f; m.add = 0.0f; m.identity = 0;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = i + seed;
        const float a0 = gen(k, 1), a1 = gen(k, 2), b0 = gen(k, 3), b1 = gen(k, 4);
        const p2::f2 q = p2::div_exact_checked(p2::mk(a0, a1), p2::mk(b0, b1));
        if (!same(q.x, a0 / b0)) bad[0]++;
        if (!same(q.y, a1 / b1)) bad[0]++;
        const float s0 = fabsf(a0), s1 = fabsf(b1);
        const p2::f2 r = p2::sqrt_exact(p2::mk(s0, s1));
        if (!same(r.x, sqrtf(s0))) bad[1]++;
        if (!same(r.y, sqrtf(s1))) bad[1]++;
        const p2::f2 t = p2::atanf2(p2::mk(a1, b0), tab);
        if (!same(t.x, gf_atanf(a1))) { bad[2]++; if (dbg) { const unsigned slot = atomicAdd(&dbg[0], 1u); if (slot < 16) { dbg[1 + slot * 4] = __float_as_uint(a1); dbg[2 + slot * 4] = __float_as_uint(t.x); dbg[3 + slot * 4] = __float_as_uint(gf_atanf(a1)); dbg[4 + slot * 4] = __float_as_uint(b0); } } }
        if (!same(t.y, gf_atanf(b0))) bad[2]++;
        // uniform divisor: typical frame sizes and random ones
        const float dv = (k & 1) ? (float)(16 + (mix(k) % 16368)) : fabsf(gen(k, 5));
        m.div = dv; m.rcp = 1.0f / dv;
        const float ad = fabsf(dv);
        m.fast_div = (ad >= 0x1p-40f && ad <= 0x1p40f) ? 1 : 0;
        if (!same(div_uniform(a0, m), a0 / dv)) bad[3]++;
        if (m.fast_div) {
            bool flagged = false;                        // the kernel sends flagged pairs to the scalar code; unflagged ones must be exact
            const p2::f2 mq = map_apply_x2(p2::mk(a0, b1), m, flagged);
            { const float n0 = fabsf(a0), n1 = fabsf(b1);      // the host-side guarantees of map_apply_x2, restated for random operands
              if (!((n0 == 0.0f || n0 > 0x1p-74f) && (n1 == 0.0f || n1 > 0x1p-74f) && dv <= 0x1p20f)) flagged = true; }
            if (!flagged && !same(mq.x, ((a0 - 0.0f) * 1.0f) / dv + 0.0f)) bad[3]++;
            if (!flagged && !same(mq.y, ((b1 - 0.0f) * 1.0f) / dv + 0.0f)) bad[3]++;
        }
        if (round_away_i32(a0) != as_i32(rs_round(a0))) bad[3]++;
        if (round_away_i32(b1 * 32.0f) != as_i32(rs_round(b1 * 32.0f))) bad[3]++;
        {   // conversion-free rounding: exact inside its window, a safe sentinel outside (contract at round_half_away_w)
            int wa, wb;
            round_half_away_w(p2::mul(p2::mk(a0, b0), p2::bc(64.0f)), wa, wb);
            const float t[2] = {a0 * 32.0f, b0 * 32.0f}; const int r[2] = {wa >> 1, wb >> 1};
            for (int j = 0; j < 2; ++j) {
                const int e = as_i32(rs_round(t[j]));
                const bool fine = (t[j] > -0.25f && t[j] < 4194304.0f) ? (r[j] == e)
                                : (t[j] >= 4194304.0f) ? (r[j] >= 4194304) : (r[j] <= 0 && (e >= 0 || r[j] < 0));   // t <= -1/4 or NaN
                if (!fine) bad[3]++;
            }
            const int lim = (int)(mix(k ^ 0x55u) & 0x3fffffu);
            int ra, rb;
            round_away_clamped_x2(p2::mk(a1, b1), lim, ra, rb);
            if (ra != max(min(as_i32(rs_round(a1)), lim), 0)) bad[3]++;
            if (rb != max(min(as_i32(rs_round(b1)), lim), 0)) bad[3]++;
        }
        // straight-line atanf on the range the kernel admits (r = sqrt(a), a in [2^-56, 2^48))
        const float c0 = fabsf(a1), c1 = fabsf(b0);
        if (in_window_r2(c0) && in_window_r2(c1)) {
            const p2::f2 rr = p2::sqrt_seq(p2::mk(c0, c1));
            if (!same(rr.x, sqrtf(c0)) || !same(rr.y, sqrtf(c1))) bad[1]++;
            const p2::f2 tc = p2::atanf2_core(rr, p2::GF_ATAN_TAB);
            if (!same(tc.x, gf_atanf(rr.x))) bad[2]++;
            if (!same(tc.y, gf_atanf(rr.y))) bad[2]++;
        }
        // unguarded division inside the windows the kernel checks
        if (p2::in_window(b0) && p2::in_window(b1) && zero_or_in_window(a0) && zero_or_in_window(a1)) {
            const p2::f2 qs = p2::div_seq(p2::mk(a0, a1), p2::mk(b0, b1));
            // a == -0 comes out as +0 (the residual fma loses the sign); no consumer in the kernel sees the sign of a zero
            const float e0 = a0 / b0, e1 = a1 / b1;
            if (!(same(qs.x, e0) || (qs.x == 0.0f && e0 == 0.0f)) || !(same(qs.y, e1) || (qs.y == 0.0f && e1 == 0.0f))) bad[0]++;
        }
    }
    for (int j = 0; j < 4; ++j) if (bad[j]) atomicAdd(&out[j], bad[j]);
}
// Exhaustive sweeps (opt-in, GF_RUN_EXHAUSTIVE=1 in the tests): every float of the packed atanf's admitted range [2^-28, 2^24) and of
// the packed square root's window [2^-56, 2^48), two consecutive floats per thread (lane .x / lane .y), against the scalar functions.
__global__ void sweep_kernel(uint32_t lo, uint32_t hi, int which, unsigned long long* out) {
    unsigned long long bad = 0;
    const uint32_t step = 2u * gridDim.x * blockDim.x;
    for (uint64_t u = (uint64_t)lo + 2u * (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x); u + 1 < hi; u += step) {
        const float a = __uint_as_float((uint32_t)u), b = __uint_as_float((uint32_t)u + 1u);
        if (which == 0) {
            const p2::f2 t = p2::atanf2_core(p2::mk(a, b), p2::GF_ATAN_TAB);
            if (!same(t.x, gf_atanf(a))) bad++;
            if (!same(t.y, gf_atanf(b))) bad++;
        } else {
            const p2::f2 r = p2::sqrt_seq(p2::mk(a, b));
            if (!same(r.x, sqrtf(a))) bad++;
            if (!same(r.y, sqrtf(b))) bad++;
        }
    }
    if (bad) atomicAdd(out, bad);
}

// Filtered pre-pass certificate (Lens2<opencv_fisheye>::approx_v) against the exact chain, on the real MUFU units: for `n_cfg` random
// configurations (fisheye coefficients of either sign up to the conditioning cap, a random mid-row matrix = K_new^-1-like scale times a
// rotation of up to ~25 degrees with random translation terms, frame sizes 1280..8192) every pixel of a sampled grid is evaluated both
// ways.  out[0] = pixels inside the regime, out[1] = pixels whose |tv_approx - tv_exact| EXCEEDS the certificate's bound (must be 0),
// out[2] = pixels the certificate calls uncertain (distance to the rounding boundary <= bound), out[3] = max |diff| / bound in 1e-6 units.
// Each configuration's lens has its own radial table (radial_table_cap, as the warp builds it); a lens whose table misses the error
// budget would run without the filter and is skipped.
struct FilterCfg { float m[9]; float k[4]; float f1, c1; int on; int w, h; };
__global__ void filter_check_kernel(const FilterCfg* __restrict__ cfgs, const float4* __restrict__ tabs, int n_cfg, int step, float rho,
                                    unsigned long long* out) {
    unsigned long long in_regime = 0, violations = 0, uncertain = 0; unsigned worst = 0;
    for (int ci = blockIdx.y; ci < n_cfg; ci += gridDim.y) {
        const FilterCfg C = cfgs[ci];
        if (!C.on) continue;
        const float4* const rtab = tabs + (size_t)ci * GF_RADIAL_ROWS;
        const FilterEps eps = filter_eps(C.c1, rho);                                  // the kernel's certificate tolerance
        gf_kernel_params P; memset(&P, 0, sizeof(P));
        for (int i = 0; i < 4; ++i) P.k[i] = C.k[i];
        P.f[0] = C.f1; P.f[1] = C.f1; P.c[0] = 0.5f * (float)C.w; P.c[1] = C.c1;
        const int nx = (C.w + step - 1) / step, ny = (C.h + step - 1) / step;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nx * ny; i += gridDim.x * blockDim.x) {
            const float px = (float)((i % nx) * step + (ci % step)), py = (float)((i / nx) * step + ((ci / 3) % step));
            const float _x = (px * C.m[0] + py * C.m[1]) + C.m[2];
            const float _y = (px * C.m[3] + py * C.m[4]) + C.m[5];
            const float _w = (px * C.m[6] + py * C.m[7]) + C.m[8];
            using L = Lens2<GF_LENS_OPENCV_FISHEYE>;
            if (!L::divisors_ok(_w, _w)) continue;                                   // the kernel's divisor test
            const float tvc = L::approx_v(_x, _y, _w, P, rtab);
            const float tv = tvc + P.c[1];
            if (!(fabsf(tv) < 0x1p20f)) continue;                                     // also r^2 at or above the cap: NaN rows
            float ex, ey;
            Lens<GF_LENS_OPENCV_FISHEYE>::distort(_x, _y, _w, P, false, ex, ey);       // the reference's arithmetic (scalar exact code)
            const float tv_exact = ey * P.f[1] + P.c[1];
            const float bound = __fmaf_rn(fabsf(tvc), eps.rel, eps.abs);
            const float diff = fabsf(tv - tv_exact);
            ++in_regime;
            if (!(diff <= bound)) ++violations;
            int row;
            if (!certify_row(tv, bound, C.h, row)) ++uncertain;
            const float ratio = bound > 0.0f ? diff / bound : (diff > 0.0f ? 1e9f : 0.0f);
            worst = max(worst, (unsigned)fminf(ratio * 1e6f, 4.0e9f));
        }
    }
    if (in_regime) atomicAdd(&out[0], in_regime);
    if (violations) atomicAdd(&out[1], violations);
    if (uncertain) atomicAdd(&out[2], uncertain);
    atomicMax(&out[3], (unsigned long long)worst);
}
} // namespace

extern "C" GF_API int gf_cuda_selftest_filter(int device, unsigned long long seed, int n_cfg, int step, unsigned long long* out4) {
    if (!out4 || n_cfg < 1 || step < 1) return GF_ERR_BAD_PARAMS;
    CK(nullptr, cudaSetDevice(device));
    std::vector<FilterCfg> cfgs((size_t)n_cfg);
    std::vector<float4> tabs((size_t)n_cfg * GF_RADIAL_ROWS);
    uint64_t st = seed * 0x9E3779B97F4A7C15ULL + 12345u;
    auto rnd = [&]() { st ^= st << 13; st ^= st >> 7; st ^= st << 17; return (double)(st >> 11) * (1.0 / 9007199254740992.0); };   // [0, 1)
    for (int i = 0; i < n_cfg; ++i) {
        FilterCfg& C = cfgs[(size_t)i];
        const int sizes[5][2] = { {3840, 2160}, {1920, 1080}, {7680, 4320}, {1280, 720}, {8192, 4320} };
        C.w = sizes[i % 5][0]; C.h = sizes[i % 5][1];
        // coefficients: scale a random sign pattern so that sum |k_i| t^(2i+2) reaches 1/4 somewhere between 0.6 and 1.55 rad
        double k[4]; for (int j = 0; j < 4; ++j) k[j] = (rnd() * 2.0 - 1.0) * pow(0.35, j);
        const double t_hit = 0.6 + 0.95 * rnd(), t2 = t_hit * t_hit;
        const double B = t2 * (fabs(k[0]) + t2 * (fabs(k[1]) + t2 * (fabs(k[2]) + t2 * fabs(k[3]))));
        const double sc = (i % 7 == 0) ? 0.02 / B : 0.25 / B;                 // every 7th: a weak lens (cap at 1.55 rad)
        for (int j = 0; j < 4; ++j) C.k[j] = (float)(k[j] * sc);
        C.on = radial_table_cap(C.k, &tabs[(size_t)i * GF_RADIAL_ROWS]) > 0.0f;
        // mid-row matrix: (K_new R)^-1 with focal length 0.3..1.2 widths and a rotation of up to ~25 degrees about a random axis
        const double f = (0.3 + 0.9 * rnd()) * C.w, cx = 0.5 * C.w, cy = 0.5 * C.h;
        double ax[3] = { rnd() - 0.5, rnd() - 0.5, rnd() - 0.5 }; const double an = sqrt(ax[0]*ax[0] + ax[1]*ax[1] + ax[2]*ax[2]) + 1e-12;
        for (double& v : ax) v /= an;
        const double ang = 0.45 * rnd(), c = cos(ang), s = sin(ang), t = 1.0 - c;
        const double R[9] = { t*ax[0]*ax[0] + c, t*ax[0]*ax[1] - s*ax[2], t*ax[0]*ax[2] + s*ax[1],
                              t*ax[0]*ax[1] + s*ax[2], t*ax[1]*ax[1] + c, t*ax[1]*ax[2] - s*ax[0],
                              t*ax[0]*ax[2] - s*ax[1], t*ax[1]*ax[2] + s*ax[0], t*ax[2]*ax[2] + c };
        // inverse of K R = R^T K^-1, K^-1 = [[1/f, 0, -cx/f], [0, 1/f, -cy/f], [0, 0, 1]]
        const double Ki[9] = { 1.0 / f, 0.0, -cx / f, 0.0, 1.0 / f, -cy / f, 0.0, 0.0, 1.0 };
        for (int r = 0; r < 3; ++r) for (int q = 0; q < 3; ++q) C.m[r * 3 + q] = (float)(R[0 * 3 + r] * Ki[0 * 3 + q] + R[1 * 3 + r] * Ki[1 * 3 + q] + R[2 * 3 + r] * Ki[2 * 3 + q]);
        C.f1 = (float)((0.3 + 0.9 * rnd()) * C.w); C.c1 = (float)(cy + (rnd() - 0.5) * 40.0);
    }
    GrowBuf<FilterCfg> d_cfg; GrowBuf<float4> d_tab; GrowBuf<unsigned long long> d_out;
    CK(nullptr, d_cfg.reserve(cfgs.size(), nullptr));
    CK(nullptr, d_tab.reserve(tabs.size(), nullptr));
    CK(nullptr, d_out.reserve(4, nullptr));
    CK(nullptr, cudaMemcpy(d_cfg.ptr, cfgs.data(), cfgs.size() * sizeof(FilterCfg), cudaMemcpyHostToDevice));
    CK(nullptr, cudaMemcpy(d_tab.ptr, tabs.data(), tabs.size() * sizeof(float4), cudaMemcpyHostToDevice));
    CK(nullptr, cudaMemset(d_out.ptr, 0, 4 * sizeof(unsigned long long)));
    filter_check_kernel<<<dim3(132, (unsigned)(n_cfg < 64 ? n_cfg : 64)), 256>>>(d_cfg.ptr, d_tab.ptr, n_cfg, step, kFilterRho, d_out.ptr);
    CK(nullptr, cudaGetLastError());
    CK(nullptr, cudaDeviceSynchronize());
    CK(nullptr, cudaMemcpy(out4, d_out.ptr, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return GF_OK;
}

namespace {
__global__ void certify_kernel(const float* __restrict__ t, size_t n, float eps, int lim, uint8_t* __restrict__ cert, int32_t* __restrict__ row) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        int r;
        cert[i] = certify_row(t[i], eps, lim, r) ? 1 : 0;
        row[i] = r;
    }
}
} // namespace

extern "C" GF_API int gf_cuda_selftest_certify(int device, const float* t, size_t n, float eps, int lim, uint8_t* cert_out, int32_t* row_out) {
    if (!t || !cert_out || !row_out) return GF_ERR_BAD_PARAMS;
    if (n == 0) return GF_OK;
    CK(nullptr, cudaSetDevice(device));
    GrowBuf<float> d_t; GrowBuf<uint8_t> d_c; GrowBuf<int32_t> d_r;
    CK(nullptr, d_t.reserve(n, nullptr)); CK(nullptr, d_c.reserve(n, nullptr)); CK(nullptr, d_r.reserve(n, nullptr));
    CK(nullptr, cudaMemcpy(d_t.ptr, t, n * sizeof(float), cudaMemcpyHostToDevice));
    certify_kernel<<<132 * 8, 256>>>(d_t.ptr, n, eps, lim, d_c.ptr, d_r.ptr);
    CK(nullptr, cudaGetLastError());
    CK(nullptr, cudaDeviceSynchronize());
    CK(nullptr, cudaMemcpy(cert_out, d_c.ptr, n, cudaMemcpyDeviceToHost));
    CK(nullptr, cudaMemcpy(row_out, d_r.ptr, n * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return GF_OK;
}

namespace {
// One CTA per group, exactly as sync_cost_kernel treats a pair: the group's keys go to shared memory (<= SYNC_SMEM_KEYS) or to global
// scratch, each thread counts its valid ones, and sync_select_add adds the group's k-smallest sum to sums[group].
__global__ void __launch_bounds__(SYNC_THREADS) sync_select_kernel(const uint32_t* __restrict__ in, const uint2* __restrict__ groups,
                                                                   uint32_t* __restrict__ scratch, unsigned long long* __restrict__ sums) {
    extern __shared__ uint32_t skeys[];
    __shared__ unsigned hist[256];
    __shared__ uint64_t red[SYNC_THREADS / 32];
    __shared__ uint32_t s_prefix, s_rank;
    const uint2 gr = groups[blockIdx.x];             // first key, key count
    if (gr.y == 0) return;
    uint32_t* keys = gr.y <= SYNC_SMEM_KEYS ? skeys : scratch + gr.x;
    uint64_t valid = 0;
    for (uint32_t i = threadIdx.x; i < gr.y; i += SYNC_THREADS) {
        const uint32_t key = in[gr.x + i];
        if (key != SYNC_NO_KEY) ++valid;
        keys[i] = key;
    }
    sync_select_add(keys, gr.y, valid, hist, red, s_prefix, s_rank, &sums[blockIdx.x]);
}
} // namespace

extern "C" GF_API int gf_cuda_selftest_sync_select(int device, const uint32_t* keys, const size_t* group_sizes, size_t n_groups,
                                                   unsigned long long* out_sums) {
    if (n_groups == 0) return GF_OK;
    if (!keys || !group_sizes || !out_sums || n_groups > 0x7fffffffu) return GF_ERR_BAD_PARAMS;
    std::vector<uint2> groups(n_groups);
    size_t total = 0, max_n = 0;
    for (size_t i = 0; i < n_groups; ++i) {
        if (group_sizes[i] > 0xFFFFFFFFu - total) return GF_ERR_BAD_PARAMS;       // offsets are 32-bit, as in sync_cost_kernel
        groups[i] = make_uint2((unsigned)total, (unsigned)group_sizes[i]);
        total += group_sizes[i];
        max_n = std::max(max_n, group_sizes[i]);
    }
    CK(nullptr, cudaSetDevice(device));
    GrowBuf<uint32_t> d_in, d_scratch; GrowBuf<uint2> d_groups; GrowBuf<unsigned long long> d_sums;
    CK(nullptr, d_in.reserve(std::max<size_t>(total, 1), nullptr));
    CK(nullptr, d_groups.reserve(n_groups, nullptr));
    CK(nullptr, d_sums.reserve(n_groups, nullptr));
    if (max_n > SYNC_SMEM_KEYS) CK(nullptr, d_scratch.reserve(total, nullptr));
    if (total) CK(nullptr, cudaMemcpy(d_in.ptr, keys, total * sizeof(uint32_t), cudaMemcpyHostToDevice));
    CK(nullptr, cudaMemcpy(d_groups.ptr, groups.data(), n_groups * sizeof(uint2), cudaMemcpyHostToDevice));
    CK(nullptr, cudaMemset(d_sums.ptr, 0, n_groups * sizeof(unsigned long long)));
    const unsigned smem = (unsigned)std::min<size_t>(max_n, SYNC_SMEM_KEYS) * (unsigned)sizeof(uint32_t);
    sync_select_kernel<<<(unsigned)n_groups, SYNC_THREADS, smem>>>(d_in.ptr, d_groups.ptr, d_scratch.ptr, d_sums.ptr);
    CK(nullptr, cudaGetLastError());
    CK(nullptr, cudaDeviceSynchronize());
    CK(nullptr, cudaMemcpy(out_sums, d_sums.ptr, n_groups * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return GF_OK;
}

// out2[0]: mismatches of atanf2_core over all floats in [2^-28, 2^24); out2[1]: of sqrt_seq over all floats in [2^-56, 2^48).
extern "C" GF_API int gf_cuda_selftest_exhaustive(int device, unsigned long long* out2) {
    if (!out2) return GF_ERR_BAD_PARAMS;
    CK(nullptr, cudaSetDevice(device));
    GrowBuf<unsigned long long> d;
    CK(nullptr, d.reserve(2, nullptr));
    CK(nullptr, cudaMemset(d.ptr, 0, 2 * sizeof(unsigned long long)));
    sweep_kernel<<<132 * 16, 256>>>(__float_as_uint_host(0x1p-28f), __float_as_uint_host(0x1p24f), 0, d.ptr);
    CK(nullptr, cudaGetLastError());
    sweep_kernel<<<132 * 16, 256>>>(__float_as_uint_host(0x1p-56f), __float_as_uint_host(0x1p48f), 1, d.ptr + 1);
    CK(nullptr, cudaGetLastError());
    CK(nullptr, cudaDeviceSynchronize());
    CK(nullptr, cudaMemcpy(out2, d.ptr, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return GF_OK;
}

extern "C" GF_API int gf_cuda_selftest(int device, unsigned long long n, unsigned long long seed, unsigned long long* out4) {
    if (!out4) return GF_ERR_BAD_PARAMS;
    CK(nullptr, cudaSetDevice(device));
    GrowBuf<unsigned long long> d;
    CK(nullptr, d.reserve(4, nullptr));
    CK(nullptr, cudaMemset(d.ptr, 0, 4 * sizeof(unsigned long long)));
    GrowBuf<uint32_t> dbg;
    if (getenv("GF_SELFTEST_DEBUG")) { dbg.reserve(65, nullptr); cudaMemset(dbg.ptr, 0, 65 * 4); }
    selftest_kernel<<<132 * 8, 256>>>(n, seed, d.ptr, dbg.ptr);
    CK(nullptr, cudaGetLastError());
    CK(nullptr, cudaDeviceSynchronize());
    CK(nullptr, cudaMemcpy(out4, d.ptr, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    if (dbg.ptr) {
        uint32_t h[65]; cudaMemcpy(h, dbg.ptr, sizeof(h), cudaMemcpyDeviceToHost);
        for (unsigned i = 0; i < (h[0] < 16 ? h[0] : 16); ++i) {
            float x, g, w, o; memcpy(&x, &h[1 + i * 4], 4); memcpy(&g, &h[2 + i * 4], 4); memcpy(&w, &h[3 + i * 4], 4); memcpy(&o, &h[4 + i * 4], 4);
            printf("atanf2 mismatch: x=%a (%08x) got=%a want=%a other-lane=%a (%08x)\n", x, h[1 + i * 4], g, w, o, h[4 + i * 4]);
        }
    }
    return GF_OK;
}
