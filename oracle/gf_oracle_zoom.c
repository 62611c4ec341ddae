/* gf_oracle_zoom.c — see gf_oracle_zoom.h.  Built with the flags of oracle/Makefile (strict IEEE, no FMA contraction). */
#include "gf_oracle_zoom.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

/* `x as usize` for f64 */
static inline size_t rs_f64_as_usize(double x) {
    if (x != x) return 0;
    if (x <= 0.0) return 0;
    if (x >= 18446744073709551616.0) return SIZE_MAX;
    return (size_t)x;
}

/* ---- zooming::calculate_fovs after find_fov (zooming/mod.rs:55-68, fov_iterative.rs:59-69, zoom_dynamic.rs:15-189) ---- */

/* get_frames_per_window — zoom_dynamic.rs:82-88 (reads the GLOBAL adaptive_zoom_window) */
static size_t get_frames_per_window(const gf_zoom_params* zp) {
    size_t frames = rs_f64_as_usize(floor(zp->adaptive_zoom_window * zp->scaled_fps));
    if (frames % 2 == 0) frames += 1;
    if (frames > ((size_t)1 << 40)) abort();                 /* the reference panics allocating the window (capacity overflow) */
    return frames;
}
/* pad_edge — :114-125 (a non-empty) */
static double* pad_edge(const double* a, size_t n, size_t pad) {
    double* p = (double*)malloc((n + 2 * pad) * sizeof(double));
    for (size_t i = 0; i < n; ++i) p[pad + i] = a[i];
    for (size_t i = 0; i < pad; ++i) { p[i] = a[0]; p[pad + n + i] = a[n - 1]; }
    return p;
}
/* gaussian_window_normalized(m, m / 6) — :102-112 */
static double* gaussian_window_normalized(size_t m) {
    double* w = (double*)calloc(m, sizeof(double));
    double std = (double)m / 6.0, sig2 = 2.0 * std * std, sum = 0.0;
    long half = (long)m / 2;
    for (long x = -half, k = 0; x <= half; ++x, ++k) w[k] = exp(-(double)(x * x) / sig2);
    for (size_t k = 0; k < m; ++k) sum += w[k];
    for (size_t k = 0; k < m; ++k) w[k] /= sum;
    return w;
}

typedef struct { double fps, window; size_t frames; long half_frames; double* gaussian_window; } data_per_timestamp;   /* :7-13 */

/* min_rolling_dynamic — :129-143 */
static void min_rolling_dynamic(const double* a, size_t alen, long max_window_half, const data_per_timestamp* d, size_t n, double* out) {
    for (size_t di = 0; di < n; ++di) {
        long i = (long)di + (max_window_half - d[di].half_frames);
        if (i >= 0 && (size_t)i + d[di].frames <= alen) {       /* the reference logs an error otherwise; every frame has the same window */
            double m = a[i];
            for (size_t j = 1; j < d[di].frames; ++j) m = fmin(m, a[i + j]);
            out[di] = m;
        }
    }
}
/* convolve_dynamic — :145-163 */
static void convolve_dynamic(const double* a, size_t alen, long max_window_half, const data_per_timestamp* d, size_t n, double* out) {
    for (size_t di = 0; di < n; ++di) {
        long i = (long)di + (max_window_half - d[di].half_frames);
        if (i >= 0 && (size_t)i + d[di].frames <= alen) {
            double s = 0.0;
            for (size_t j = 0; j < d[di].frames; ++j) s += a[i + j] * d[di].gaussian_window[j];
            out[di] = s;
        }
    }
}
/* envelope_follower — :165-189; alpha < 0 stands for None: each frame's 1 - exp(-(1 / fps) / window) */
static void envelope_follower_dynamic(const double* a, size_t n, const data_per_timestamp* d, double alpha, double* out) {
    double* alphas = (double*)malloc(n * sizeof(double));
    double* rev = (double*)malloc(n * sizeof(double));
    for (size_t i = 0; i < n; ++i) alphas[i] = alpha >= 0.0 ? alpha : 1.0 - exp(-(1.0 / d[i].fps) / d[i].window);
    double q = a[n - 1];
    for (size_t r = 0; r < n; ++r) { size_t i = n - 1 - r; double x = a[i]; q = fmin(x, x * alphas[i] + q * (1.0 - alphas[i])); rev[r] = q; }
    q = rev[n - 1];
    for (size_t r = 0; r < n; ++r) { double x = rev[n - 1 - r]; q = fmin(x, x * alphas[r] + q * (1.0 - alphas[r])); out[r] = q; }
    free(alphas); free(rev);
}

void gf_oracle_zoom_fovs(const gf_zoom_params* zp, const double* fov_values, const double* window, const double* speed,
                         int zooming_keyed, int speed_keyed, size_t n, double* out_fovs, double* out_minimal_fovs) {
    if (n == 0) return;                                                          /* zooming/mod.rs:36-38 */
    double* v = (double*)malloc(n * sizeof(double));
    memcpy(v, fov_values, n * sizeof(double));
    if (zp->n_trim_ranges > 0) {                                                 /* fov_iterative.rs:59-69 */
        double l = (double)(n - 1);
        double max_fov = v[0];
        for (size_t i = 1; i < n; ++i) max_fov = fmax(max_fov, v[i]);
        for (size_t i = 0; i < n; ++i) {
            int within = 0;
            for (size_t r = 0; r < zp->n_trim_ranges; ++r)
                if (i >= rs_f64_as_usize(floor(l * zp->trim_ranges[2 * r])) && i <= rs_f64_as_usize(ceil(l * zp->trim_ranges[2 * r + 1]))) within = 1;
            if (!within) v[i] = max_fov;
        }
    }
    memcpy(out_minimal_fovs, v, n * sizeof(double));                             /* fov_minimal = fov_values.clone() (mod.rs:57, zoom_dynamic.rs:18) */
    if (zp->adaptive_zoom_window < -0.9) {                                       /* static zoom, mod.rs:55-61 */
        double m = v[0];
        for (size_t i = 1; i < n; ++i) m = fmin(m, v[i]);
        for (size_t i = 0; i < n; ++i) out_fovs[i] = m;
    } else if (zp->adaptive_zoom_window > 0.0001) {                              /* dynamic zoom, mod.rs:62-64 */
        int envelope = zp->adaptive_zoom_method == 1;                            /* ZoomMethod::from: anything else is the gaussian filter */
        if (zooming_keyed || (zp->video_speed_affects_zooming && (zp->video_speed != 1.0 || speed_keyed))) {   /* zoom_dynamic.rs:22-55 */
            data_per_timestamp* d = (data_per_timestamp*)malloc(n * sizeof(data_per_timestamp));
            size_t max_window = 0;
            for (size_t i = 0; i < n; ++i) {
                double w = window[i];
                if (zp->video_speed_affects_zooming) w *= fabs(speed[i]);
                size_t frames = get_frames_per_window(zp);
                if (frames > max_window) max_window = frames;
                d[i].window = w; d[i].fps = zp->scaled_fps; d[i].frames = frames; d[i].half_frames = (long)(frames / 2);
                d[i].gaussian_window = gaussian_window_normalized(frames);
            }
            if (!envelope) {
                size_t mwh = max_window / 2;
                double* pad = pad_edge(v, n, mwh);
                double* mn = (double*)malloc(n * sizeof(double));
                min_rolling_dynamic(pad, n + 2 * mwh, (long)mwh, d, n, mn);
                free(pad);
                pad = pad_edge(mn, n, mwh);
                convolve_dynamic(pad, n + 2 * mwh, (long)mwh, d, n, out_fovs);
                free(pad); free(mn);
            } else {
                double second_pass_alpha = 1.0 - exp(-(1.0 / zp->scaled_fps) / 0.2);
                double* tmp = (double*)malloc(n * sizeof(double));
                envelope_follower_dynamic(v, n, d, -1.0, tmp);
                envelope_follower_dynamic(tmp, n, d, second_pass_alpha, out_fovs);
                free(tmp);
            }
            for (size_t i = 0; i < n; ++i) free(d[i].gaussian_window);
            free(d);
        } else {
            gf_oracle_zoom_dynamic(v, n, zp->adaptive_zoom_window, zp->scaled_fps, envelope, out_fovs);   /* :56-76 */
        }
    } else {                                                                     /* zoom disabled, mod.rs:65-67 */
        for (size_t i = 0; i < n; ++i) out_fovs[i] = 1.0;
    }
    free(v);
}

void gf_oracle_calculate_fovs(const gf_compute_params* cp, const gf_zoom_params* zp, int model, int digital,
                              const double* timestamps_ms, const double* window, const double* speed, int zooming_keyed, int speed_keyed,
                              size_t n, double* out_fovs, double* out_minimal_fovs) {
    if (n == 0) return;
    gf_compute_params c = *cp;                                                   /* zooming/mod.rs:40-49 */
    c.fov_scale = 1.0; c.n_fovs = 0; c.n_minimal_fovs = 0; c.output_width = c.width; c.output_height = c.height;
    double* fov_values = (double*)malloc(n * sizeof(double));
    for (size_t i = 0; i < n; ++i)
        fov_values[i] = gf_oracle_find_fov(&c, model, digital, cp->output_width, cp->output_height, zp->fov_algorithm_margin, timestamps_ms[i], i);
    gf_oracle_zoom_fovs(zp, fov_values, window, speed, zooming_keyed, speed_keyed, n, out_fovs, out_minimal_fovs);
    free(fov_values);
}
