// sync_select.cuh — the k-smallest sum of the visual-features sync cost (visual_features.rs:69-82), one CTA per group of keys.
// sync_cost_kernel (zoom_kernel.cu) runs it on the keys of one (candidate, pair); gf_cuda_selftest_sync_select (selftest.cu) on raw
// keys from the host, so that the selection can be checked on keys the point path rarely produces.
#pragma once
#include <cstdint>

namespace gf {

constexpr int SYNC_THREADS = 256;
constexpr unsigned SYNC_SMEM_KEYS = 8192;       // distance keys per pair held in shared memory; larger pairs keep them in global scratch
constexpr uint32_t SYNC_NO_KEY = 0xFFFFFFFFu;   // a point pair outside the frame; every real key is <= 2^31 (frames of <= 32768 px a side)

__device__ __forceinline__ uint64_t block_sum_u64(uint64_t v, uint64_t* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();                            // `red` may still be read from the previous reduction
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    uint64_t s = 0;
    for (int w = 0; w < SYNC_THREADS / 32; ++w) s += red[w];
    return s;
}

// keys[0 .. n): this thread wrote keys[threadIdx.x + j * SYNC_THREADS] and counts `valid` of them below SYNC_NO_KEY.  With m the CTA's
// count of valid keys and k = (m as f64 * 0.9) as usize, finds the k-th smallest key T by radix select (one 256-bin histogram per byte,
// high byte first) and adds sum(keys < T) + (k - count(keys < T)) * T — the sum of the k smallest — to *sum with an integer atomic, whose
// order does not matter.  NO_KEY sorts above every valid key and k < m, so T is always a valid key.  The shared arguments are the CTA's.
__device__ __forceinline__ void sync_select_add(const uint32_t* keys, uint32_t n, uint64_t valid, unsigned* hist, uint64_t* red,
                                                uint32_t& s_prefix, uint32_t& s_rank, unsigned long long* sum) {
    const uint64_t m = block_sum_u64(valid, red);
    const uint64_t k = (uint64_t)((double)m * 0.9);     // (len as f64 * 0.9) as usize
    if (k == 0) return;
    if (threadIdx.x == 0) { s_prefix = 0; s_rank = (uint32_t)k; }
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int b = threadIdx.x; b < 256; b += SYNC_THREADS) hist[b] = 0;
        __syncthreads();                                 // also publishes s_prefix / s_rank and (first pass) every key
        const uint32_t prefix = s_prefix, hi = shift == 24 ? 0u : (0xFFFFFFFFu << (shift + 8));
        for (uint32_t i = threadIdx.x; i < n; i += SYNC_THREADS) {
            const uint32_t key = keys[i];
            if ((key & hi) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x < 32) {                          // one warp: lane l scans bins 8l..8l+7
            const int l = threadIdx.x;
            unsigned c[8], own = 0;
            for (int j = 0; j < 8; ++j) { c[j] = hist[8 * l + j]; own += c[j]; }
            unsigned incl = own;
            for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xffffffffu, incl, o); if (l >= o) incl += t; }
            const uint32_t rank = s_rank;
            unsigned before = incl - own;
            if (before < rank && rank <= incl) {         // exactly one lane holds the bin of the rank-th key
                int j = 0;
                while (before + c[j] < rank) before += c[j++];
                s_rank = rank - before;
                s_prefix = prefix | ((uint32_t)(8 * l + j) << shift);
            }
        }
        __syncthreads();                                 // the scan has read `hist` before the next pass clears it
    }
    const uint32_t T = s_prefix;
    uint64_t below = 0, n_below = 0;
    for (uint32_t i = threadIdx.x; i < n; i += SYNC_THREADS) {
        const uint32_t key = keys[i];
        if (key < T) { below += key; ++n_below; }
    }
    below = block_sum_u64(below, red);
    n_below = block_sum_u64(n_below, red);
    if (threadIdx.x == 0) atomicAdd(sum, (unsigned long long)(below + (k - n_below) * (uint64_t)T));
}

} // namespace gf
