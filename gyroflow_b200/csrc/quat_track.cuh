// quat_track.cuh — quaternion tracks (TimeQuat = BTreeMap<i64 us, UnitQuaternion<f64>>, src/core/gyro_source/mod.rs:34) as sorted
// arrays, and the lookups the per-frame producers need.  Shared by frame_transform.cu (FrameTransform::at_timestamp) and
// zoom_kernel.cu (at_timestamp_for_points) through frame_geometry.cuh; host and device compile the same functions.
//
//   qslerp             nalgebra 0.34.2 UnitQuaternion::slerp (shortest arc; `a` when the quaternions coincide)
//   sync_offset_at     GyroSource::offset_at_timestamp         gyro_source/mod.rs:884-909
//   quat_at_timestamp  GyroSource::quat_at_timestamp           gyro_source/mod.rs:857-879
#pragma once
#include <cstdint>
#include <cstddef>
#include <cmath>

#define GF_QT_HD __host__ __device__ __forceinline__

namespace gf {

struct Quat { double w, i, j, k; };

GF_QT_HD Quat qmul(const Quat& a, const Quat& b) {      // Hamilton product
    return { a.w * b.w - a.i * b.i - a.j * b.j - a.k * b.k,
             a.w * b.i + a.i * b.w + a.j * b.k - a.k * b.j,
             a.w * b.j - a.i * b.k + a.j * b.w + a.k * b.i,
             a.w * b.k + a.i * b.j - a.j * b.i + a.k * b.w };
}
GF_QT_HD Quat qinv(const Quat& a) { return { a.w, -a.i, -a.j, -a.k }; }     // unit quaternion: conjugate

GF_QT_HD Quat qslerp(const Quat& a, Quat b, double t) {
    double d = a.w * b.w + a.i * b.i + a.j * b.j + a.k * b.k;
    if (d < 0.0) { b = { -b.w, -b.i, -b.j, -b.k }; d = -d; }
    if (d >= 1.0) return a;
    const double hang = acos(d);
    const double s = sqrt(1.0 - d * d);
    if (fabs(s) < 1e-14) return a;          // nalgebra would report an ambiguous configuration; neighbours on a track never are
    const double ta = sin((1.0 - t) * hang) / s, tb = sin(t * hang) / s;
    return { a.w * ta + b.w * tb, a.i * ta + b.i * tb, a.j * ta + b.j * tb, a.k * ta + b.k * tb };
}

// offsets / offsets_adjusted: BTreeMap<i64 us, f64 ms> as sorted arrays.  n == 0: the scalar fallback (a single sync point).
struct SyncOffsets { const int64_t* ts; const double* ms; size_t n; double scalar_ms; };

// gyro_source/mod.rs:884-909 — 0 points: the scalar offset (gyro_offset_ms); 1 point: its value; else linear interpolation between the neighbours of
// clamp(ts, first + 1, last - 1), with the fraction taken from the UNclamped timestamp (so it extrapolates outside the range).
GF_QT_HD double sync_offset_at(const SyncOffsets& o, double timestamp_ms) {
    if (o.n == 0) return o.scalar_ms;
    if (o.n == 1) return o.ms[0];
    const int64_t first_ts = o.ts[0], last_ts = o.ts[o.n - 1];
    const double us = timestamp_ms * 1000.0;                     // `as i64`: truncating, saturating, NaN -> 0
    const int64_t timestamp_us = us != us ? 0 : (us >= 9.2233720368547758e18 ? INT64_MAX : (us <= -9.2233720368547758e18 ? INT64_MIN : (int64_t)us));
    int64_t lookup = timestamp_us;
    if (lookup > last_ts - 1) lookup = last_ts - 1;              // .min(last_ts - 1).max(first_ts + 1)
    if (lookup < first_ts + 1) lookup = first_ts + 1;
    size_t lo = 0, hi = o.n;                                     // last key <= lookup (exists: lookup >= first + 1)
    while (hi - lo > 1) { const size_t mid = (lo + hi) / 2; if (o.ts[mid] <= lookup) lo = mid; else hi = mid; }
    if (o.ts[lo] == lookup) return o.ms[lo];
    if (lo + 1 >= o.n) return 0.0;                               // range(lookup..) empty: falls through to the final 0.0
    const double time_delta = (double)(o.ts[lo + 1] - o.ts[lo]);
    const double fract = (double)(timestamp_us - o.ts[lo]) / time_delta;
    return o.ms[lo] + (o.ms[lo + 1] - o.ms[lo]) * fract;
}

struct Track { const int64_t* ts; const double* q; size_t n; };
GF_QT_HD Quat track_at(const Track& tr, size_t idx) { const double* p = tr.q + idx * 4; return { p[0], p[1], p[2], p[3] }; }

// f64::round (half away from zero) then `as i64`
GF_QT_HD int64_t round_to_i64(double v) { return (int64_t)llround(v); }

GF_QT_HD Quat quat_at_timestamp(const Track& tr, double duration_ms, const SyncOffsets& offsets, double timestamp_ms) {
    if (tr.n < 2 || duration_ms <= 0.0) return { 1.0, 0.0, 0.0, 0.0 };
    timestamp_ms -= sync_offset_at(offsets, timestamp_ms);       // :859
    const int64_t first_ts = tr.ts[0], last_ts = tr.ts[tr.n - 1];
    int64_t lookup = round_to_i64(timestamp_ms * 1000.0);
    if (lookup > last_ts) lookup = last_ts;
    if (lookup < first_ts) lookup = first_ts;
    size_t lo = 0, hi = tr.n;                                    // invariant: ts[lo] <= lookup < ts[hi] (hi may be n)
    while (hi - lo > 1) { const size_t mid = (lo + hi) / 2; if (tr.ts[mid] <= lookup) lo = mid; else hi = mid; }
    if (tr.ts[lo] == lookup) return track_at(tr, lo);
    if (lo + 1 >= tr.n) return track_at(tr, lo);
    const double time_delta = (double)(tr.ts[lo + 1] - tr.ts[lo]);
    const double fract = (double)(lookup - tr.ts[lo]) / time_delta;
    return qslerp(track_at(tr, lo), track_at(tr, lo + 1), fract);
}

// CatmullRom<Vector3<f64>>::interpolate — gyro_source/splines.rs:22-83.  Points as two arrays: positions[n], values[n][3].
// Returns false for None (fewer than two points, NaN, t outside [first, last)).
struct Spline3 { const double* pos; const double* val; size_t n; };
GF_QT_HD bool catmull_rom3(const Spline3& s, double t, double (&out)[3]) {
    if (s.n < 2 || t != t) return false;
    // binary_search_by: Ok(i) for an exact hit, Err(i) = insertion point
    size_t lo = 0, hi = s.n; bool exact = false; size_t hit = 0;
    while (lo < hi) {
        const size_t mid = lo + (hi - lo) / 2;
        if (s.pos[mid] == t) { exact = true; hit = mid; break; }
        if (s.pos[mid] < t) lo = mid + 1; else hi = mid;
    }
    size_t lower;
    if (exact) { if (hit == s.n - 1) return false; lower = hit; }
    else { if (lo >= s.n || lo == 0) return false; lower = lo - 1; }
    if (lower + 1 >= s.n) return false;
    const double* a = s.val + 3 * lower; const double* b = s.val + 3 * (lower + 1);
    const double k = (t - s.pos[lower]) / (s.pos[lower + 1] - s.pos[lower]);
    for (int c = 0; c < 3; ++c) {
        const double x = lower == 0 ? a[c] * 2.0 - b[c] : s.val[3 * (lower - 1) + c];
        const double y = lower + 2 >= s.n ? b[c] * 2.0 - a[c] : s.val[3 * (lower + 2) + c];
        // ((((a * 3 - x) - b * 3) + y) * 0.5) * t*t*t + ((b - x) * 0.5) * t + a + (((b * 4 + a * -5 + x + x) - y) * 0.5) * t*t   (:76-81)
        out[c] = ((((a[c] * 3.0 - x) - b[c] * 3.0) + y) * 0.5) * k * k * k
               + ((b[c] - x) * 0.5) * k
               + a[c]
               + (((b[c] * 4.0 + a[c] * -5.0 + x + x) - y) * 0.5) * k * k;
    }
    return true;
}

} // namespace gf
