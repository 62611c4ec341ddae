/* gf_oracle_optsync.c — CPU oracle of the automatic sync-point choice (TEST INFRASTRUCTURE; never linked into the product).
 *
 * A literal C transcription of the exact stages of OptimSync (src/core/synchronization/optimsync.rs): `new`'s resampling (:30-66),
 * `blackman` (:15-27) with glibc cosf, and the part of `run` after the spectra (:117-223): rank, masks, the NMS double loop and the
 * segments' max_by fold.  The spectra themselves have no exact oracle: tests/np_optsync.py takes them in f64 (scipy.fft).
 * Built by optsync.mk with the flags of oracle/Makefile (strict IEEE, no FMA contraction). */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

/* `x as usize` for f64 (saturating, NaN 0) */
static size_t f64_as_usize(double x) {
    if (x != x || x <= 0.0) return 0;
    if (x >= 18446744073709551616.0) return SIZE_MAX;
    return (size_t)x;
}

/* OptimSync::new (:30-66).  gyro is n x 3, has_gyro (NULL: every sample has a gyro reading) marks `gyro.is_some()`.  Returns the number
 * of resampled samples; *sample_rate receives avg_sr and out (NULL: count only) the resampled gyro, n_res x 3.  n must be >= 1. */
size_t gf_oracle_optsync_resample(const double* ts, const double* gyro, const uint8_t* has_gyro, size_t n, double* sample_rate, double* out) {
    const double duration_ms = ts[n - 1] - ts[0];
    size_t samples_total = 0;
    for (size_t i = 0; i < n; ++i) samples_total += has_gyro ? (has_gyro[i] != 0) : 1;
    const double avg_sr = (double)samples_total / duration_ms * 1000.0;
    *sample_rate = avg_sr;
    const size_t n_res = f64_as_usize(duration_ms * avg_sr / 1000.0);
    if (!out) return n_res;
    for (size_t i = 0; i < n_res; ++i) {
        const double t = (double)i * 1000.0 / avg_sr;
        /* raw_imu.partition_point(|s| s.timestamp_ms < t): the timestamps are sorted, so a lower-bound search finds the same index */
        size_t lo = 0, hi = n;
        while (lo < hi) { const size_t mid = lo + (hi - lo) / 2; if (ts[mid] < t) lo = mid + 1; else hi = mid; }
        const size_t i_r = lo < n - 1 ? lo : n - 1;
        const size_t i_l = (i_r > 1 ? i_r : 1) - 1;
        double l[3] = {0, 0, 0}, r[3] = {0, 0, 0};                     /* unwrap_or_default */
        if (!has_gyro || has_gyro[i_l]) for (int j = 0; j < 3; ++j) l[j] = gyro[i_l * 3 + j];
        if (!has_gyro || has_gyro[i_r]) for (int j = 0; j < 3; ++j) r[j] = gyro[i_r * 3 + j];
        for (int j = 0; j < 3; ++j) {
            if (i_l == i_r) out[i * 3 + j] = l[j];
            else out[i * 3 + j] = (l[j] * (ts[i_r] - t) + r[j] * (t - ts[i_l])) / (ts[i_r] - ts[i_l]);
        }
    }
    return n_res;
}

/* blackman (:15-27), f32 with std::f32::consts::PI and f32::cos = cosf */
void gf_oracle_optsync_blackman(size_t width, float* out) {
    const float a0 = 7938.0f / 18608.0f, a1 = 9240.0f / 18608.0f, a2 = 1430.0f / 18608.0f;
    const float pi = 3.14159265358979323846f;
    const float size = (float)(width - 1);
    for (size_t i = 0; i < width; ++i) {
        const float n = (float)i;
        out[i] = a0 - a1 * cosf(2.0f * pi * n / size) + a2 * cosf(4.0f * pi * n / size);
    }
}

static float nlfunc(float arg, float trip_point) { return arg < trip_point ? 0.0f : arg - trip_point; }

/* run (:117-223) from the merged band energies on: bands is n_win x (lf, mf, hf), trim_ranges_s n_trim x (start, end).  rank receives
 * rank_clone (n_win floats), *ratio 16 / sample_rate, points_ms at most `target` sync points; returns their number. */
size_t gf_oracle_optsync_select(const float* bands, size_t n_win, double sample_rate, size_t fft_size, size_t target,
                                const double* trim_ranges_s, size_t n_trim, double* points_ms, float* rank_out, double* ratio_out,
                                float* rank, float* rank_nms /* n_win floats each, scratch */) {
    const size_t step_size_samples = 16;
    const size_t nms_radius = f64_as_usize((sample_rate / 16.0 / 2.0) * 8.0);
    float mf_max = 0.0f;
    for (size_t i = 0; i < n_win; ++i) mf_max = fmaxf(mf_max, bands[i * 3 + 1]);
    const int low_motion = mf_max < 50.0f;
    for (size_t i = 0; i < n_win; ++i) {
        const float lf = bands[i * 3], mf = bands[i * 3 + 1], hf = bands[i * 3 + 2];
        if (low_motion) rank[i] = (lf + mf) / (1.0f + nlfunc(hf, 450.0f) * 0.003f);
        else rank[i] = mf / (1.0f + nlfunc(hf, 450.0f) * 0.003f) / (1.0f + nlfunc(lf, 650.0f) * 0.003f);
        rank_out[i] = rank[i];
    }
    const double ratio = (double)step_size_samples / sample_rate;
    *ratio_out = ratio;
    for (size_t i = 0; i < n_win; ++i) {
        const double time = (double)i * ratio;
        int any = 0;
        for (size_t k = 0; k < n_trim; ++k) any |= time >= trim_ranges_s[2 * k] && time <= trim_ranges_s[2 * k + 1];
        if (rank[i] < 50.0f || !any) rank[i] = 0.0f;
    }
    const double total_duration = (double)n_win * ratio;
    if (total_duration > 12.0) {
        for (size_t i = 0; i < n_win; ++i) {
            const double time = (double)i * ratio;
            if (time < 2.0 || time >= (total_duration - 2.0)) rank[i] = 0.0f;
        }
    }
    for (size_t i = 0; i < n_win; ++i) rank_nms[i] = rank[i];
    for (size_t i = 0; i < n_win; ++i) {
        const int64_t lo = (int64_t)i - (int64_t)nms_radius;
        const size_t hi = i + nms_radius < n_win - 1 ? i + nms_radius : n_win - 1;
        for (size_t j = lo > 0 ? (size_t)lo : 0; j < hi; ++j)
            if (rank[j] < rank[i]) rank_nms[j] = 0.0f;
    }
    const size_t segment_size = (n_win + target - 1) / target;
    size_t n_points = 0;
    for (size_t s = 0; s < target; ++s) {
        const size_t start = s * segment_size;
        const size_t end = start + segment_size < n_win ? start + segment_size : n_win;
        if (start >= end) continue;                   /* get(start..end) is None, or the slice is empty: max_by gives None */
        /* max_by(partial_cmp, NaN -> Equal): fold from the first element, the next one wins unless the kept one compares Greater */
        size_t best = start;
        for (size_t j = start + 1; j < end; ++j)
            if (!(rank_nms[best] > rank_nms[j])) best = j;
        const float value = rank_nms[best];
        if (value < 0.1f) continue;
        points_ms[n_points++] = ((double)best * (double)step_size_samples + (double)fft_size / 2.0) / sample_rate * 1000.0;
    }
    return n_points;
}
