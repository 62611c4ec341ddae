// filter_prepass.cu — the host side of the packed fisheye kernel's filtered rolling-shutter pre-pass (Lens2<opencv_fisheye>::approx_v).
#include <cstring>
#include <cmath>
#include <algorithm>
#include "warp_kernel.cuh"
#include "c_abi_internal.h"

using namespace gf;
namespace {

// The deferred-pair queue holds this many pairs (4 MB: a quarter of a 4K frame's pairs); a pair that finds it full is rendered inline by
// the main launch.  The tail launch has kTailThreadsPerSM threads (16 blocks of the packed kernel's 32 x 4) per multiprocessor.
constexpr unsigned kDeferCap = 1u << 20;
constexpr unsigned kTailThreadsPerSM = 2048;

// The certificate |tv_approx - tv_exact| <= (rho + 2^-22) |tv - c_y| + 2^-22 |c_y| assumes that the polynomial s = 1 + k0 t^2 + k1 t^4 +
// k2 t^6 + k3 t^8 stays within [3/4, 5/4] (its rounding error and its sensitivity to the error of t are then bounded,
// profiles/FILTER_ANALYSIS.md): a_cap = tan^2(t_cap) with t_cap the largest angle (<= 1.55 rad) for which sum |k_i| t^(2i+2) <= 1/4.
// Returns 0 when the lens is too strongly curved for the filter to be worth it (t_cap < 0.5 rad).
float filter_a_cap(const float* k) {
    auto B = [&](double t) { const double t2 = t * t; return t2 * (fabs((double)k[0]) + t2 * (fabs((double)k[1]) + t2 * (fabs((double)k[2]) + t2 * fabs((double)k[3])))); };
    for (int i = 0; i < 4; ++i) if (!std::isfinite(k[i])) return 0.0f;
    double lo = 0.0, hi = 1.55;
    if (B(hi) > 0.25) { for (int it = 0; it < 60; ++it) { const double mid = 0.5 * (lo + hi); if (B(mid) <= 0.25) lo = mid; else hi = mid; } }
    else lo = hi;
    if (lo < 0.5) return 0.0f;
    const double a = tan(lo) * tan(lo);
    return (float)std::min(a * 0.999, 16000.0);                 // stay inside the table (r^2 < 2^14) and below the exact bound
}

// T(a) = atan(sqrt a) / sqrt a in f64
double radial_T(double a) { const double r = sqrt(a); return r < 1e-4 ? 1.0 - a / 3.0 + a * a / 5.0 : atan(r) / r; }
// What every lens's table shares, computed once for the fitted rows: the intervals, T at their Chebyshev nodes, and the check points
// with T there
struct RadialGrid {
    static constexpr int N = GF_RADIAL_FIT_ROWS, kChk = 65;     // 64 steps per interval, both ends included
    double lo[N], hi[N], h[N];
    double node_a[N][4], node_T[N][4];
    double chk_a[N][kChk], chk_T[N][kChk];
    double vinv[4][4];              // inverse of the Vandermonde matrix of the nodes 1 + t_q, t_q = cos((2q + 1) pi / 8), in units of h
    RadialGrid() {
        double t[4], V[4][8];
        for (int q = 0; q < 4; ++q) t[q] = cos((2 * q + 1) * 3.14159265358979323846 / 8.0);
        for (int r = 0; r < 4; ++r) for (int c = 0; c < 8; ++c) V[r][c] = c < 4 ? pow(1.0 + t[r], c) : (c - 4 == r ? 1.0 : 0.0);
        for (int c = 0; c < 4; ++c) {               // Gauss-Jordan with partial pivoting
            int p = c;
            for (int r = c + 1; r < 4; ++r) if (fabs(V[r][c]) > fabs(V[p][c])) p = r;
            for (int j = 0; j < 8; ++j) std::swap(V[c][j], V[p][j]);
            const double d = V[c][c];
            for (int j = 0; j < 8; ++j) V[c][j] /= d;
            for (int r = 0; r < 4; ++r) if (r != c) { const double f = V[r][c]; for (int j = 0; j < 8; ++j) V[r][j] -= f * V[c][j]; }
        }
        for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) vinv[r][c] = V[r][c + 4];
        for (int i = 0; i < N; ++i) {
            const int e = i / 16, j = i % 16;
            lo[i] = ldexp(1.0 + j / 16.0, e - 30); hi[i] = ldexp(1.0 + (j + 1) / 16.0, e - 30);
            h[i] = 0.5 * (hi[i] - lo[i]);
            for (int q = 0; q < 4; ++q) { node_a[i][q] = lo[i] + h[i] * (1.0 + t[q]); node_T[i][q] = radial_T(node_a[i][q]); }
            for (int q = 0; q < kChk; ++q) { chk_a[i][q] = (double)(float)(lo[i] + (hi[i] - lo[i]) * q / 64.0); chk_T[i][q] = radial_T(chk_a[i][q]); }
        }
    }
};

// R(a) = T(a) s(theta) with theta^2 = a T(a)^2 and s = 1 + k0 theta^2 + ... + k3 theta^8, one cubic c0 + d (c1 + d (c2 + d c3)) in
// d = a - lo per 1/16-octave interval [lo, hi) of a over [2^-30, 2^14), fitted in f64 at the interval's four Chebyshev nodes and rounded
// to f32.  The rows below 2^-30 repeat the first fitted row (R changes by less than 2^-29 relative there); a_cap is rounded down to an
// interval boundary, and the rows from there on hold NaN, up to the last of the GF_RADIAL_ROWS bit patterns.  Every fitted row is
// checked on 65 points: the f32 coefficients' cubic, evaluated in f64, must stay within kRadialBudget (relative) of R, the table error
// of profiles/FILTER_ANALYSIS.md step 3.  Returns the rounded a_cap, or 0 when some row misses the budget (or a_cap is 0).
float build_radial_table(const float* k, float a_cap, float4* rows) {
    static const RadialGrid* const G = new RadialGrid();
    constexpr double kRadialBudget = 0x1p-23;
    uint32_t cap_bits; memcpy(&cap_bits, &a_cap, 4);
    const int n_valid = std::max(0, std::min(GF_RADIAL_FIT_ROWS, (int)(cap_bits >> 19) - GF_RADIAL_FIT));
    const double k0 = k[0], k1 = k[1], k2 = k[2], k3 = k[3];
    auto R = [&](double a, double T) { const double q = a * T * T; return T * (1.0 + q * (k0 + q * (k1 + q * (k2 + q * k3)))); };
    bool ok = n_valid > 0;
    for (int i = 0; i < GF_RADIAL_ROWS; ++i) rows[i] = make_float4(NAN, NAN, NAN, NAN);
    for (int i = 0; i < n_valid; ++i) {
        double f[4], c[4];
        for (int q = 0; q < 4; ++q) f[q] = R(G->node_a[i][q], G->node_T[i][q]);
        for (int r = 0; r < 4; ++r) c[r] = G->vinv[r][0] * f[0] + G->vinv[r][1] * f[1] + G->vinv[r][2] * f[2] + G->vinv[r][3] * f[3];
        const double hh = G->h[i];
        const float4 row = make_float4((float)c[0], (float)(c[1] / hh), (float)(c[2] / (hh * hh)), (float)(c[3] / (hh * hh * hh)));
        rows[GF_RADIAL_FIT + i] = row;
        for (int q = 0; q < RadialGrid::kChk; ++q) {
            const double a = G->chk_a[i][q], d = a - G->lo[i];
            const double v = row.x + d * (row.y + d * (row.z + d * (double)row.w));
            const double want = R(a, G->chk_T[i][q]);
            if (!(fabs(v - want) <= kRadialBudget * fabs(want))) ok = false;
        }
    }
    for (int i = 0; i < GF_RADIAL_FIT; ++i) rows[i] = rows[GF_RADIAL_FIT];
    uint32_t r_bits = cap_bits & 0xfff80000u; float a_cap_r; memcpy(&a_cap_r, &r_bits, 4);
    return ok ? a_cap_r : 0.0f;
}

} // namespace

float gf::radial_table_cap(const float* k, float4* rows) { return build_radial_table(k, filter_a_cap(k), rows); }

int FilterPrepass::table(const float* k, cudaStream_t st, std::string* err, const Table** out) {
    uint32_t key[4]; memcpy(key, k, sizeof(key));
    Table *t = nullptr, *lru = &tables[0];
    for (Table& e : tables) {
        if (e.last_use && memcmp(e.key, key, sizeof(key)) == 0) t = &e;
        if (e.last_use < lru->last_use) lru = &e;
    }
    if (!t) {
        t = lru; t->last_use = 0;
        if (!t->done) CK(err, create_event(t->done));
        CK(err, cudaEventSynchronize(t->done.get()));          // every frame that read this entry has finished
        CK(err, t->h.reserve(GF_RADIAL_ROWS, st)); CK(err, t->d.reserve(GF_RADIAL_ROWS, st));
        t->a_cap = radial_table_cap(k, t->h.ptr); builds++;
        CK(err, cudaMemcpyAsync(t->d.ptr, t->h.ptr, GF_RADIAL_ROWS * sizeof(float4), cudaMemcpyHostToDevice, st));
        CK(err, cudaEventRecord(t->done.get(), st));
        memcpy(t->key, key, sizeof(key));
    }
    t->last_use = ++uses;
    *out = t->a_cap > 0.0f ? t : nullptr;
    return GF_OK;
}

int FilterPrepass::launch(KernelFn fn, dim3 grid, dim3 block, WarpArgs& A, const Table& t, cudaStream_t st, std::string* err,
                          unsigned long long& launches) {
    if (!queue.ptr) {
        CK(err, queue.reserve(kDeferCap, st)); CK(err, counts.reserve(2, st));
        CK(err, cudaMemsetAsync(counts.ptr, 0, 2 * sizeof(unsigned), st));
    }
    const unsigned cur = (unsigned)(frames++ & 1ull);
    A.feat |= F_FILTER;
    A.flt.q = queue.ptr; A.flt.cap = (uint32_t)queue.len;
    A.flt.count = counts.ptr + cur; A.flt.count_next = counts.ptr + (cur ^ 1u);
    A.flt.mid_row = A.matrices + (size_t)(A.p.matrix_count / 2) * GF_MATRIX_STRIDE;
    const FilterEps eps = filter_eps(A.p.c[1]);                      // |c_y| >= 2^-10 without F_WILD
    A.flt.rtab = t.d.ptr; A.flt.eps_rel = eps.rel; A.flt.eps_abs = eps.abs;
    A.flt.tail = 0;
    CK(err, launch_pdl(fn, grid, block, A, st));
    CK(err, cudaEventRecord(t.done.get(), st));    // the tail launch runs the exact pre-pass and does not read the table
    A.flt.tail = 1;                                // the deferred pairs, exact pre-pass; also re-arms the other counter
    // one thread per deferred pair for up to 2 % of a 4K frame's pairs in a single wave of tiny blocks (idle blocks exit at once); more
    // entries than threads are covered by the grid-stride loop
    CK(err, launch_pdl(fn, dim3(sm_count * kTailThreadsPerSM / (block.x * block.y)), block, A, st));
    launches++;
    return GF_OK;
}

int FilterPrepass::stats(cudaStream_t st, std::string* err, uint64_t* out6) const {
    unsigned count = 0;
    if (frames > 0) {
        CK(err, cudaMemcpyAsync(&count, counts.ptr + ((frames - 1) & 1ull), sizeof(count), cudaMemcpyDeviceToHost, st));
        CK(err, cudaStreamSynchronize(st));
    }
    out6[0] = frames; out6[1] = count; out6[2] = kDeferCap; out6[3] = (uint64_t)sm_count * kTailThreadsPerSM;
    out6[4] = builds; out6[5] = uses - builds;
    return GF_OK;
}
