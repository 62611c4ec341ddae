// optimal_sync.cu — the automatic choice of sync points: OptimSync::new and OptimSync::run (src/core/synchronization/optimsync.rs:30-225),
// which Stabilization::get_optimal_sync_points (src/core/lib.rs:2043-2065) runs for autosync.
//
// Device: the resampling of `new` (resample_kernel, bit for bit) and, per window of `run`, the three band energies of the merged
// half-spectra (band_kernel: Bluestein over a power-of-two Stockham FFT in shared memory, f32; nothing per bin leaves the CTA).
// Host: `new`'s sizes and refusals (os_sizes) and the rest of `run`: rank, masks, an O(windows) NMS and the segments (os_select).
#include <cmath>
#include <vector>

#include "c_abi_internal.h"

using namespace gf;

namespace {

constexpr size_t kStep = 16;                 // step_size_samples (:80)
constexpr size_t kMaxN = 8192;               // fft_size cap: Bluestein's M = 2^ceil(log2(2N - 1)) <= 16384 complex f32 = 128 KB of smem
constexpr unsigned kMaxM = 16384;
constexpr unsigned kMaxThreads = 1024;
constexpr unsigned kMaxBfly = kMaxM / 2 / kMaxThreads;   // butterflies per thread and FFT stage
constexpr size_t kWindowsPerLaunch = size_t(1) << 24;

// `x as usize` for f64 (saturating, NaN 0)
size_t f64_as_usize(double x) {
    if (x != x || x <= 0.0) return 0;
    if (x >= 18446744073709551616.0) return SIZE_MAX;
    return (size_t)x;
}

struct Sizes { double sample_rate; size_t fft_size, n_resampled, n_windows; };

// OptimSync::new's arithmetic (:34-36, :54) and run's fft_size (:82), with every case the reference panics on refused.
int os_sizes(const double* ts, const uint8_t* has_gyro, size_t n, Sizes& s) {
    if (n == 0) return fail(nullptr, GF_ERR_NO_DATA, "optimal sync: empty gyro log (OptimSync::new returns None)");
    if (!ts) return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync: timestamps_ms is NULL");
    size_t count = 0;
    for (size_t i = 0; i < n; ++i) {
        if (ts[i] != ts[i]) return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync: timestamp " + std::to_string(i) + " is NaN");
        if (i && ts[i] < ts[i - 1]) return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync: timestamps decrease at " + std::to_string(i));
        count += has_gyro ? (has_gyro[i] != 0) : 1;
    }
    const double duration_ms = ts[n - 1] - ts[0];
    if (duration_ms == 0.0) return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync: the log spans no time (the sample rate is not finite)");
    const double avg_sr = (double)count / duration_ms * 1000.0;
    const double N = std::round(avg_sr);     // f64::round: half away from zero
    if (!(N >= 4.0)) return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync: FFT size round(sample rate) below 4");
    if (N > (double)kMaxN) return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync: FFT size round(sample rate) above 8192");
    s.sample_rate = avg_sr;
    s.fft_size = (size_t)N;
    s.n_resampled = f64_as_usize(duration_ms * avg_sr / 1000.0);
    s.n_windows = s.n_resampled >= s.fft_size ? (s.n_resampled - s.fft_size) / kStep + 1 : 0;   // windows(N).step_by(16)
    return GF_OK;
}

float nlfunc(float arg, float trip_point) { return arg < trip_point ? 0.0f : arg - trip_point; }   // :227-233

// run (:117-223) after the spectra, in the reference's f32 / f64 operations.  rank receives rank_clone; returns the number of points.
size_t os_select(const float* bands, size_t n_win, double sample_rate, size_t fft_size, size_t target, const double* trim, size_t n_trim,
                 double* points_ms, float* rank_out, double* ratio_out) {
    const size_t nms_radius = f64_as_usize((sample_rate / 16.0 / 2.0) * 8.0);        // :81
    float mf_max = 0.0f;                                                              // :141-142, fold(0.0, f32::max)
    for (size_t i = 0; i < n_win; ++i) mf_max = fmaxf(mf_max, bands[i * 3 + 1]);
    const bool low_motion = mf_max < 50.0f;
    std::vector<float> rank(n_win), nms(n_win);
    for (size_t i = 0; i < n_win; ++i) {                                              // :144-155
        const float lf = bands[i * 3], mf = bands[i * 3 + 1], hf = bands[i * 3 + 2];
        rank[i] = low_motion ? (lf + mf) / (1.0f + nlfunc(hf, 450.0f) * 0.003f)
                             : mf / (1.0f + nlfunc(hf, 450.0f) * 0.003f) / (1.0f + nlfunc(lf, 650.0f) * 0.003f);
        if (rank_out) rank_out[i] = rank[i];
    }
    const double ratio = (double)kStep / sample_rate;                                 // :159
    if (ratio_out) *ratio_out = ratio;
    const double total = (double)n_win * ratio;
    for (size_t i = 0; i < n_win; ++i) {                                              // :160-176
        const double time = (double)i * ratio;
        bool any = false;
        for (size_t k = 0; k < n_trim && !any; ++k) any = time >= trim[2 * k] && time <= trim[2 * k + 1];
        if (rank[i] < 50.0f || !any) rank[i] = 0.0f;
        if (total > 12.0 && (time < 2.0 || time >= total - 2.0)) rank[i] = 0.0f;
    }
    // NMS (:178-185): for j in [max(0, i - r), min(i + r, len - 1)), rank_nms[j] = 0 when rank[j] < rank[i].  So window j < len - 1 is
    // zeroed when some rank[i], i in (j - r, j + r] within the log, exceeds it; NaN neither suppresses nor is suppressed.  A monotonic
    // deque of the window's non-NaN ranks gives that maximum in O(windows).
    for (size_t i = 0; i < n_win; ++i) nms[i] = rank[i];
    if (nms_radius > 0 && n_win > 1) {
        std::vector<size_t> dq(n_win);
        size_t head = 0, tail = 0, next = 0;
        for (size_t j = 0; j + 1 < n_win; ++j) {
            const size_t hi = std::min(n_win - 1, j + nms_radius), lo = j + 1 > nms_radius ? j + 1 - nms_radius : 0;
            for (; next <= hi; ++next) {
                const float v = rank[next];
                if (v != v) continue;
                while (tail > head && rank[dq[tail - 1]] <= v) --tail;
                dq[tail++] = next;
            }
            while (tail > head && dq[head] < lo) ++head;
            if (tail > head && rank[j] < rank[dq[head]]) nms[j] = 0.0f;
        }
    }
    // segments (:187-211): the max of each by max_by(partial_cmp, NaN -> Equal), which keeps the LAST of equal elements
    size_t n_points = 0;
    const size_t seg = (n_win + target - 1) / target;
    for (size_t s = 0; s < target; ++s) {
        const size_t start = s * seg, end = std::min(start + seg, n_win);
        if (start >= end) continue;
        size_t best = start;
        for (size_t j = start + 1; j < end; ++j)
            if (!(nms[best] > nms[j])) best = j;
        if (nms[best] < 0.1f) continue;
        points_ms[n_points++] = ((double)best * (double)kStep + (double)fft_size / 2.0) / sample_rate * 1000.0;
    }
    return n_points;
}

// ---- device ----

// interp_gyro (:38-51) at ts = i * 1000 / avg_sr for each output sample i; out is axis-major (3 x n_res), cast to f32 as run does (:73-76).
__global__ void resample_kernel(const double* __restrict__ ts, const double* __restrict__ gyro, const uint8_t* __restrict__ has_gyro,
                                size_t n, double avg_sr, size_t n_res, float* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_res) return;
    const double t = (double)i * 1000.0 / avg_sr;
    size_t lo = 0, hi = n;                                    // partition_point(|s| s.timestamp_ms < t) over sorted timestamps
    while (lo < hi) { const size_t mid = lo + (hi - lo) / 2; if (ts[mid] < t) lo = mid + 1; else hi = mid; }
    const size_t i_r = lo < n - 1 ? lo : n - 1, i_l = (i_r > 1 ? i_r : 1) - 1;
    const bool hl = !has_gyro || has_gyro[i_l], hr = !has_gyro || has_gyro[i_r];     // unwrap_or_default
    for (int j = 0; j < 3; ++j) {
        const double l = hl ? gyro[i_l * 3 + j] : 0.0, r = hr ? gyro[i_r * 3 + j] : 0.0;
        const double v = i_l == i_r ? l : (l * (ts[i_r] - t) + r * (t - ts[i_l])) / (ts[i_r] - ts[i_l]);
        out[(size_t)j * n_res + i] = (float)v;
    }
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// In-place forward FFT of M = 2^L points in shared memory: radix-2 Stockham (natural order in and out).  Each stage reads the thread's
// butterflies into registers, waits, and writes them to their autosorted places; tw[t] = exp(-2 pi i t / M), t < M / 2.
__device__ void fft_smem(float2* buf, unsigned M, unsigned L, const float2* __restrict__ tw) {
    const unsigned half = M >> 1, nb = (half + blockDim.x - 1) / blockDim.x;
    for (unsigned s = 0; s < L; ++s) {
        float2 a[kMaxBfly], b[kMaxBfly];
#pragma unroll
        for (unsigned q = 0; q < kMaxBfly; ++q)
            if (q < nb) {
                const unsigned j = threadIdx.x + q * blockDim.x;
                if (j < half) { a[q] = buf[j]; b[q] = buf[j + half]; }
            }
        __syncthreads();
        const unsigned ns = 1u << s;
#pragma unroll
        for (unsigned q = 0; q < kMaxBfly; ++q)
            if (q < nb && threadIdx.x + q * blockDim.x < half) {
                const unsigned j = threadIdx.x + q * blockDim.x, k = j & (ns - 1);
                const float2 t = cmul(b[q], __ldg(tw + (k << (L - 1 - s))));     // exp(-2 pi i k / (2 ns))
                const unsigned o = ((j >> s) << (s + 1)) + k;
                buf[o] = make_float2(a[q].x + t.x, a[q].y + t.y);
                buf[o + ns] = make_float2(a[q].x - t.x, a[q].y - t.y);
            }
        __syncthreads();
    }
}

struct BandArgs {
    const float* gyro; size_t n_res;         // resampled gyro, 3 x n_res
    const float* win;                        // blackman(N)
    const float2* chirp;                     // c[n] = exp(-i pi n^2 / N), n < N
    const float2* filt;                      // FFT_M(conj(c) wrapped) / M
    const float2* tw;                        // exp(-2 pi i t / M), t < M / 2
    unsigned N, M, L, b2, b30, b2000;        // map_to_bin(2), (30), (2000); map_to_bin(0) is 0
    float scale;                             // sqrt(1 / N) / N * 256 (:83)
    size_t w0;                               // first window of the launch
    float* bands;                            // n_windows x (lf, mf, hf)
};

// One CTA per window: for each axis, the DFT of gyro * blackman by Bluestein, then |X[k] + X[N-1-k]| * scale summed over the three
// bands (:88-139).  Band energy is linear in the bins, so the axes' bins go into the same three sums.
__global__ void __launch_bounds__(kMaxThreads) band_kernel(const BandArgs A) {
    extern __shared__ float2 buf[];
    __shared__ float red[32][3];
    const size_t w = A.w0 + blockIdx.x;
    float acc[3] = {0.0f, 0.0f, 0.0f};
    for (int axis = 0; axis < 3; ++axis) {
        const float* x = A.gyro + (size_t)axis * A.n_res + w * kStep;
        for (unsigned n = threadIdx.x; n < A.M; n += blockDim.x) {
            float2 v = make_float2(0.0f, 0.0f);
            if (n < A.N) {
                const float xw = x[n] * __ldg(A.win + n);                      // zip(chunk, &win).map(|(x, y)| x * y)
                const float2 c = __ldg(A.chirp + n);
                v = make_float2(xw * c.x, xw * c.y);
            }
            buf[n] = v;
        }
        __syncthreads();
        fft_smem(buf, A.M, A.L, A.tw);
        for (unsigned k = threadIdx.x; k < A.M; k += blockDim.x) {           // conj(A * B / M): the next FFT is the inverse, conjugated
            const float2 p = cmul(buf[k], __ldg(A.filt + k));
            buf[k] = make_float2(p.x, -p.y);
        }
        __syncthreads();
        fft_smem(buf, A.M, A.L, A.tw);
        for (unsigned k = threadIdx.x; k < A.b2000; k += blockDim.x) {       // X[k] = c[k] * conj(buf[k]); bins [0, map_to_bin(2000))
            const unsigned m = A.N - 1 - k;                                   // zip(iter, iter.rev()): bin k pairs with N-1-k
            const float2 yk = buf[k], ym = buf[m];
            const float2 xk = cmul(__ldg(A.chirp + k), make_float2(yk.x, -yk.y));
            const float2 xm = cmul(__ldg(A.chirp + m), make_float2(ym.x, -ym.y));
            const float v = hypotf(xk.x + xm.x, xk.y + xm.y) * A.scale;
            acc[k < A.b2 ? 0 : (k < A.b30 ? 1 : 2)] += v;
        }
        __syncthreads();
    }
    for (int b = 0; b < 3; ++b)
        for (int o = 16; o > 0; o >>= 1) acc[b] += __shfl_down_sync(0xffffffffu, acc[b], o);
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = (blockDim.x + 31) >> 5;
    if (lane == 0) for (int b = 0; b < 3; ++b) red[warp][b] = acc[b];
    __syncthreads();
    if (threadIdx.x == 0) {
        float s[3] = {0.0f, 0.0f, 0.0f};
        for (unsigned q = 0; q < n_warps; ++q) for (int b = 0; b < 3; ++b) s[b] += red[q][b];
        for (int b = 0; b < 3; ++b) A.bands[w * 3 + b] = s[b];
    }
}

// sin and cos of pi * x in f64, x reduced to [-1/4, 1/4] around a multiple of 1/2 first, so the phase keeps f64 accuracy
void sincospi_f64(double x, double* s, double* c) {
    const double q = std::nearbyint(2.0 * x), r = x - 0.5 * q;        // x = q / 2 + r, |r| <= 1/4, exact
    const double sr = std::sin(M_PI * r), cr = std::cos(M_PI * r);
    switch (((long long)q % 4 + 4) % 4) {
    case 0: *s = sr; *c = cr; break;
    case 1: *s = cr; *c = -sr; break;
    case 2: *s = -sr; *c = -cr; break;
    default: *s = -cr; *c = sr; break;
    }
}

// In-place radix-2 FFT in f64 (host), for the Bluestein filter
void fft_f64(std::vector<double>& re, std::vector<double>& im) {
    const size_t M = re.size();
    for (size_t i = 1, j = 0; i < M; ++i) {
        size_t bit = M >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) { std::swap(re[i], re[j]); std::swap(im[i], im[j]); }
    }
    for (size_t len = 2; len <= M; len <<= 1)
        for (size_t k = 0; k < len / 2; ++k) {
            double ws, wc;
            sincospi_f64(-2.0 * (double)k / (double)len, &ws, &wc);
            for (size_t i = k; i < M; i += len) {
                const size_t j = i + len / 2;
                const double tr = re[j] * wc - im[j] * ws, ti = re[j] * ws + im[j] * wc;
                re[j] = re[i] - tr; im[j] = im[i] - ti;
                re[i] += tr; im[i] += ti;
            }
        }
}

// blackman (:15-27) on the host with libm's cosf, in f32 like the reference
void blackman(size_t width, float* out) {
    const float a0 = 7938.0f / 18608.0f, a1 = 9240.0f / 18608.0f, a2 = 1430.0f / 18608.0f;
    const float pi = 3.14159265358979323846f, size = (float)(width - 1);
    for (size_t i = 0; i < width; ++i) {
        const float n = (float)i;
        out[i] = a0 - a1 * cosf(2.0f * pi * n / size) + a2 * cosf(4.0f * pi * n / size);
    }
}

// map_to_bin (:113-119)
unsigned map_to_bin(size_t N, double sample_rate, double freq) {
    return (unsigned)std::min(std::max(std::round((double)N / sample_rate * freq), 0.0), (double)(N / 2 - 1));
}

// Upload the log and resample it into d_res (3 x n_res floats) on `st`.
struct Upload { GrowBuf<double> ts, gyro; GrowBuf<uint8_t> has; };
int resample(const double* ts, const double* gyro, const uint8_t* has_gyro, size_t n, const Sizes& s, Upload& up, GrowBuf<float>& d_res,
             cudaStream_t st) {
    CK(nullptr, up.ts.reserve(n, st));
    CK(nullptr, up.gyro.reserve(n * 3, st));
    CK(nullptr, d_res.reserve(std::max<size_t>(s.n_resampled * 3, 1), st));
    CK(nullptr, cudaMemcpyAsync(up.ts.ptr, ts, n * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(nullptr, cudaMemcpyAsync(up.gyro.ptr, gyro, n * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    if (has_gyro) {
        CK(nullptr, up.has.reserve(n, st));
        CK(nullptr, cudaMemcpyAsync(up.has.ptr, has_gyro, n, cudaMemcpyHostToDevice, st));
    }
    if (s.n_resampled) {
        const unsigned threads = 256;
        resample_kernel<<<(unsigned)((s.n_resampled + threads - 1) / threads), threads, 0, st>>>(
            up.ts.ptr, up.gyro.ptr, has_gyro ? up.has.ptr : nullptr, n, s.sample_rate, s.n_resampled, d_res.ptr);
        CK(nullptr, cudaGetLastError());
    }
    return GF_OK;
}

int check_log(const double* ts, const double* gyro, const uint8_t* has_gyro, size_t n, Sizes& s) {
    const int rc = os_sizes(ts, has_gyro, n, s);
    if (rc != GF_OK) return rc;
    if (!gyro) return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync: gyro_xyz is NULL");
    // the resampled gyro is indexed by 32-bit grids and by size_t (3 x n_res floats): far beyond any log
    if (s.n_resampled > (size_t(1) << 36)) return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync: too many resampled samples");
    return GF_OK;
}

}  // namespace

extern "C" GF_API int gf_optimal_sync_sizes(const double* timestamps_ms, const uint8_t* has_gyro, size_t n, double* sample_rate,
                                            size_t* fft_size, size_t* n_resampled, size_t* n_windows) {
    Sizes s{};
    const int rc = os_sizes(timestamps_ms, has_gyro, n, s);
    if (rc != GF_OK) return rc;
    if (sample_rate) *sample_rate = s.sample_rate;
    if (fft_size) *fft_size = s.fft_size;
    if (n_resampled) *n_resampled = s.n_resampled;
    if (n_windows) *n_windows = s.n_windows;
    return GF_OK;
}

extern "C" GF_API int gf_optimal_sync_select(const float* bands, size_t n_windows, double sample_rate, size_t fft_size, size_t target,
                                             const double* trim_ranges_s, size_t n_trim, double* points_ms, size_t* n_points, float* rank,
                                             double* ratio) {
    if (target == 0) return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync: target_sync_points is 0");
    if ((n_windows && !bands) || (n_trim && !trim_ranges_s) || !points_ms || !n_points)
        return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync select: NULL array");
    *n_points = os_select(bands, n_windows, sample_rate, fft_size, target, trim_ranges_s, n_trim, points_ms, rank, ratio);
    return GF_OK;
}

extern "C" GF_API int gf_cuda_selftest_optimal_sync_resample(int device, const double* timestamps_ms, const double* gyro_xyz,
                                                             const uint8_t* has_gyro, size_t n, float* out, size_t n_out) {
    Sizes s{};
    const int rc = check_log(timestamps_ms, gyro_xyz, has_gyro, n, s);
    if (rc != GF_OK) return rc;
    if (n_out != s.n_resampled || (n_out && !out))
        return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync resample: out must hold 3 x n_resampled floats");
    if (!n_out) return GF_OK;
    CK(nullptr, cudaSetDevice(device));
    Upload up; GrowBuf<float> d_res;
    const int r2 = resample(timestamps_ms, gyro_xyz, has_gyro, n, s, up, d_res, nullptr);
    if (r2 != GF_OK) return r2;
    CK(nullptr, cudaMemcpy(out, d_res.ptr, s.n_resampled * 3 * sizeof(float), cudaMemcpyDeviceToHost));
    return GF_OK;
}

extern "C" GF_API int gf_cuda_optimal_sync_points(int device, const double* timestamps_ms, const double* gyro_xyz, const uint8_t* has_gyro,
                                                  size_t n, size_t target, const double* trim_ranges_s, size_t n_trim, double* points_ms,
                                                  size_t* n_points, float* rank, float* bands, double* ratio, void* cu_stream) {
    if (target == 0) return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync: target_sync_points is 0");
    if ((n_trim && !trim_ranges_s) || !points_ms || !n_points) return fail(nullptr, GF_ERR_BAD_PARAMS, "optimal sync: NULL array");
    Sizes s{};
    const int rc = check_log(timestamps_ms, gyro_xyz, has_gyro, n, s);
    if (rc != GF_OK) return rc;
    std::vector<float> h_bands(s.n_windows * 3);
    if (s.n_windows) {
        const size_t N = s.fft_size;
        unsigned L = 0;
        while ((1u << L) < 2 * N - 1) ++L;
        const unsigned M = 1u << L, threads = std::min(kMaxThreads, std::max(32u, M / 2));   // whole warps
        // Bluestein's chirp c[n] = exp(-i pi n^2 / N), its phase from n^2 mod 2N, and the filter FFT_M(b) / M with b[m] = conj(c[m]) for
        // m < N and b[M - m] = conj(c[m]) for 0 < m < N, built in f64 and stored as f32
        std::vector<float2> chirp(N), filt(M), tw(M / 2);
        std::vector<double> bre(M, 0.0), bim(M, 0.0);
        for (size_t m = 0; m < N; ++m) {
            double sn, cs;
            sincospi_f64(-(double)((uint64_t)m * m % (2 * (uint64_t)N)) / (double)N, &sn, &cs);
            chirp[m] = make_float2((float)cs, (float)sn);
            bre[m] = cs; bim[m] = -sn;
            if (m) { bre[M - m] = cs; bim[M - m] = -sn; }
        }
        fft_f64(bre, bim);
        for (unsigned k = 0; k < M; ++k) filt[k] = make_float2((float)(bre[k] / M), (float)(bim[k] / M));
        for (unsigned t = 0; t < M / 2; ++t) {
            double sn, cs;
            sincospi_f64(-2.0 * (double)t / (double)M, &sn, &cs);
            tw[t] = make_float2((float)cs, (float)sn);
        }
        std::vector<float> win(N);
        blackman(N, win.data());

        const cudaStream_t st = (cudaStream_t)cu_stream;
        CK(nullptr, cudaSetDevice(device));
        Upload up; GrowBuf<float> d_res, d_win, d_bands; GrowBuf<float2> d_chirp, d_filt, d_tw;
        const int r2 = resample(timestamps_ms, gyro_xyz, has_gyro, n, s, up, d_res, st);
        if (r2 != GF_OK) return r2;
        CK(nullptr, d_win.reserve(N, st));
        CK(nullptr, d_chirp.reserve(N, st));
        CK(nullptr, d_filt.reserve(M, st));
        CK(nullptr, d_tw.reserve(M / 2, st));
        CK(nullptr, d_bands.reserve(s.n_windows * 3, st));
        CK(nullptr, cudaMemcpyAsync(d_win.ptr, win.data(), N * sizeof(float), cudaMemcpyHostToDevice, st));
        CK(nullptr, cudaMemcpyAsync(d_chirp.ptr, chirp.data(), N * sizeof(float2), cudaMemcpyHostToDevice, st));
        CK(nullptr, cudaMemcpyAsync(d_filt.ptr, filt.data(), M * sizeof(float2), cudaMemcpyHostToDevice, st));
        CK(nullptr, cudaMemcpyAsync(d_tw.ptr, tw.data(), M / 2 * sizeof(float2), cudaMemcpyHostToDevice, st));
        const unsigned smem = M * (unsigned)sizeof(float2);
        CK(nullptr, cudaFuncSetAttribute(band_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kMaxM * sizeof(float2))));
        BandArgs A{d_res.ptr, s.n_resampled, d_win.ptr, d_chirp.ptr, d_filt.ptr, d_tw.ptr, (unsigned)N, M, L,
                   map_to_bin(N, s.sample_rate, 2.0), map_to_bin(N, s.sample_rate, 30.0), map_to_bin(N, s.sample_rate, 2000.0),
                   std::sqrt(1.0f / (float)N) / (float)N * 256.0f, 0, d_bands.ptr};
        for (size_t w0 = 0; w0 < s.n_windows; w0 += kWindowsPerLaunch) {
            A.w0 = w0;
            band_kernel<<<(unsigned)std::min(kWindowsPerLaunch, s.n_windows - w0), threads, smem, st>>>(A);
            CK(nullptr, cudaGetLastError());
        }
        CK(nullptr, cudaMemcpyAsync(h_bands.data(), d_bands.ptr, s.n_windows * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(nullptr, cudaStreamSynchronize(st));
        if (bands) std::copy(h_bands.begin(), h_bands.end(), bands);
    }
    *n_points = os_select(h_bands.data(), s.n_windows, s.sample_rate, s.fft_size, target, trim_ranges_s, n_trim, points_ms, rank, ratio);
    return GF_OK;
}
