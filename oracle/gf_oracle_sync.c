/* gf_oracle_sync.c — see gf_oracle_sync.h.  Built with the flags of oracle/Makefile (strict IEEE, no FMA contraction). */
#include "gf_oracle_sync.h"

#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

/* `x as usize` for f64 */
static size_t f64_as_usize(double x) {
    if (x != x || x <= 0.0) return 0;
    if (x >= 18446744073709551616.0) return SIZE_MAX;
    return (size_t)x;
}
/* `x as isize` for f64 */
static int64_t f64_as_isize(double x) {
    if (x != x) return 0;
    if (x <= -9223372036854775808.0) return INT64_MIN;
    if (x >= 9223372036854775808.0) return INT64_MAX;
    return (int64_t)x;
}
/* `x as u64` for f32 */
static uint64_t f32_as_u64(float x) {
    if (x != x || x <= 0.0f) return 0;
    if (x >= 18446744073709551616.0f) return UINT64_MAX;
    return (uint64_t)x;
}
/* frame_at_timestamp (lib.rs:2069) `as usize`: round half away from zero, `as i32` (saturating, NaN 0), then sign-extended */
static size_t frame_at_timestamp(double timestamp_ms, double fps) {
    double r = round(timestamp_ms * (fps / 1000.0));
    int32_t i = r != r ? 0 : (r <= -2147483648.0 ? INT32_MIN : (r >= 2147483647.0 ? INT32_MAX : (int32_t)r));
    return (size_t)(int64_t)i;
}
static int cmp_u64(const void* a, const void* b) {
    uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
    return x < y ? -1 : (x > y ? 1 : 0);
}

/* undistort_points_with_rolling_shutter(pts, timestamp_ms, None, params, 1.0, false) — cpu_undistort.rs:636-641 */
static void undistort_points_rs(const gf_compute_params* params, int model, int digital, double fps, const float* pts, size_t n,
                                double timestamp_ms, float* out) {
    gf_oracle_undistort_points_rs_ex(params, model, digital, pts, n, timestamp_ms, frame_at_timestamp(timestamp_ms, fps), 1.0, 0, out);
}

/* calculate_distance — visual_features.rs:46-84 */
static double calculate_distance(const gf_compute_params* params_arg, int model, int digital, double fps, const gf_sync_pair* matched_points,
                                 size_t n_pairs, double offs, int has_rs, double rs) {
    double total_dist = 0.0;
    gf_compute_params params2 = *params_arg;
    if (has_rs) params2.frame_readout_time = rs;
    const gf_compute_params* params_ref = &params2;
    const int w = params_ref->width, h = params_ref->height;
    for (size_t p = 0; p < n_pairs; ++p) {
        const gf_sync_pair* mp = &matched_points[p];
        double timestamp_ms = (double)mp->ts_us / 1000.0;
        double timestamp_ms2 = (double)mp->next_ts_us / 1000.0;
        size_t n = mp->n;
        if (n == 0) continue;                                    /* undistort_points_with_rolling_shutter of nothing is nothing */
        float* undistorted_points1 = (float*)malloc(2 * n * sizeof(float));
        float* undistorted_points2 = (float*)malloc(2 * n * sizeof(float));
        undistort_points_rs(params_ref, model, digital, fps, mp->pts1, n, timestamp_ms - offs, undistorted_points1);
        undistort_points_rs(params_ref, model, digital, fps, mp->pts2, n, timestamp_ms2 - offs, undistorted_points2);
        uint64_t* distances = (uint64_t*)malloc(n * sizeof(uint64_t));
        size_t len = 0;
        for (size_t i = 0; i < n; ++i) {
            float p1x = undistorted_points1[2 * i], p1y = undistorted_points1[2 * i + 1];
            float p2x = undistorted_points2[2 * i], p2y = undistorted_points2[2 * i + 1];
            if (p1x > 0.0f && p1x < (float)w && p1y > 0.0f && p1y < (float)h &&
                p2x > 0.0f && p2x < (float)w && p2y > 0.0f && p2y < (float)h) {
                float dist = ((p2x - p1x) * (p2x - p1x)) + ((p2y - p1y) * (p2y - p1y));
                distances[len++] = f32_as_u64(dist);
            }
        }
        qsort(distances, len, sizeof(uint64_t), cmp_u64);
        /* only 90 % of the lines: the longest are often wrong matches */
        size_t keep = f64_as_usize((double)len * 0.9);
        for (size_t i = 0; i < keep; ++i) total_dist += (double)distances[i];
        free(distances); free(undistorted_points1); free(undistorted_points2);
    }
    return total_dist;
}

typedef struct {
    const gf_compute_params* params; int model, digital; double fps; const gf_sync_pair* pairs; size_t n_pairs;
    const double* offs; const double* rs; size_t begin, end; double* out;
} job;

static void* worker(void* arg) {
    const job* j = (const job*)arg;
    for (size_t c = j->begin; c < j->end; ++c)
        j->out[c] = calculate_distance(j->params, j->model, j->digital, j->fps, j->pairs, j->n_pairs, j->offs ? j->offs[c] : 0.0,
                                       j->rs != NULL, j->rs ? j->rs[c] : 0.0);
    return NULL;
}

/* the costs of n candidates, shared out over `threads` threads */
static void eval_candidates(const gf_compute_params* params, int model, int digital, double fps, const gf_sync_pair* pairs, size_t n_pairs,
                            const double* offs, const double* rs, size_t n, int threads, double* out) {
    size_t nt = threads > 0 ? (size_t)threads : (size_t)gf_oracle_online_cpus();
    if (nt < 1) nt = 1;
    if (nt > n) nt = n;
    if (nt <= 1) {
        job j = { params, model, digital, fps, pairs, n_pairs, offs, rs, 0, n, out };
        worker(&j);
        return;
    }
    pthread_t* th = (pthread_t*)calloc(nt, sizeof(pthread_t));
    job* jobs = (job*)calloc(nt, sizeof(job));
    for (size_t t = 0; t < nt; ++t) {
        job j = { params, model, digital, fps, pairs, n_pairs, offs, rs, n * t / nt, n * (t + 1) / nt, out };
        jobs[t] = j;
        pthread_create(&th[t], NULL, worker, &jobs[t]);
    }
    for (size_t t = 0; t < nt; ++t) pthread_join(th[t], NULL);
    free(th); free(jobs);
}

void gf_oracle_sync_costs(const gf_compute_params* cp, int model, int digital, double scaled_fps, const gf_sync_pair* pairs, size_t n_pairs,
                          const double* offsets_ms, const double* readout_ms, size_t n_candidates, int clear_offsets, int threads, double* out_costs) {
    gf_compute_params params = *cp;
    if (clear_offsets) params.gyro_offset_ms = 0.0;               /* params.gyro.write().clear_offsets() (:12-15) */
    eval_candidates(&params, model, digital, scaled_fps, pairs, n_pairs, offsets_ms, readout_ms, n_candidates, threads, out_costs);
}

/* find_min folded over the candidates in order (reduce_with(find_min), :87): `if a.1 < b.1 { a } else { b }` */
static size_t find_min(const double* cost, size_t n) {
    size_t lowest = 0;
    for (size_t i = 1; i < n; ++i) lowest = cost[lowest] < cost[i] ? lowest : i;
    return lowest;
}

size_t gf_oracle_find_sync_offsets(const gf_compute_params* cp, int model, int digital, double scaled_fps, double initial_offset_ms,
                                   double search_size_ms, int for_rs, const gf_sync_range* ranges, size_t n_ranges, int threads,
                                   gf_sync_result* out) {
    gf_compute_params params = *cp;                              /* :11-15 */
    if (!for_rs) params.gyro_offset_ms = 0.0;
    size_t n_out = 0;
    const double fps = scaled_fps;
    for (size_t r = 0; r < n_ranges; ++r) {
        const gf_sync_range* range = &ranges[r];
        const int64_t from_ts = range->from_us, to_ts = range->to_us;
        size_t n_coarse = 0;
        double* coarse;
        if (for_rs) {                                             /* estimate rolling shutter (:91-116) */
            double max_rs = 1000.0 / fps;
            int64_t steps = f64_as_isize(max_rs);
            n_coarse = steps > 0 ? (size_t)(2 * steps) : 0;
            if (n_coarse > ((size_t)1 << 32)) abort();           /* far beyond any test's job */
            coarse = (double*)calloc(n_coarse ? n_coarse : 1, sizeof(double));
            for (int64_t i = -steps, k = 0; i < steps; ++i, ++k) coarse[k] = (double)i;
        } else {                                                  /* offsets (:117-143) */
            size_t steps = f64_as_usize(search_size_ms);
            n_coarse = steps;
            if (n_coarse > ((size_t)1 << 32)) abort();
            coarse = (double*)calloc(n_coarse ? n_coarse : 1, sizeof(double));
            for (size_t i = 0; i < steps; ++i) coarse[i] = initial_offset_ms + (-(search_size_ms / 2.0) + (double)i);
        }
        if (n_coarse == 0) { free(coarse); continue; }            /* reduce_with of nothing is None: no entry */
        double* cost = (double*)malloc(n_coarse * sizeof(double));
        eval_candidates(&params, model, digital, fps, range->pairs, range->n_pairs, for_rs ? NULL : coarse, for_rs ? coarse : NULL,
                        n_coarse, threads, cost);
        double lowest0 = coarse[find_min(cost, n_coarse)];
        double fine[200], cost2[200];
        for (int i = 0; i < 200; ++i) fine[i] = lowest0 - 1.0 + ((double)i * 0.01);      /* then refine to 0.01 ms */
        eval_candidates(&params, model, digital, fps, range->pairs, range->n_pairs, for_rs ? NULL : fine, for_rs ? fine : NULL, 200, threads, cost2);
        size_t b = find_min(cost2, 200);
        if (for_rs) {
            gf_sync_result res = { 0.0, fine[b], cost2[b] };
            out[n_out++] = res;
        } else {
            double middle_timestamp = ((double)from_ts + (double)(int64_t)((uint64_t)to_ts - (uint64_t)from_ts) / 2.0) / 1000.0;
            /* only offsets within 90 % of the search size */
            if (fabs(fine[b] - initial_offset_ms) < search_size_ms * 0.9) {
                gf_sync_result res = { middle_timestamp, fine[b], cost2[b] };
                out[n_out++] = res;
            }
        }
        free(cost); free(coarse);
    }
    return n_out;
}
