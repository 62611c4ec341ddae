// zoom_kernel.cu — adaptive-zoom companion: per-frame minimal FOV by warping the frame edge (SURVEY §8 a17).
//
// Behavioural source: FovIterative::find_fov / nearest_edge / points_around_rect / interpolate_points
// (src/core/zooming/fov_iterative.rs:91-189), undistort_points_with_rolling_shutter + undistort_points
// (src/core/stabilization/cpu_undistort.rs:636-858, with the IBIS / OIS shifts and the distorting mesh), FrameTransform::at_timestamp_for_points
// (src/core/stabilization/frame_transform.rs:352-438), calculate_fovs (src/core/zooming/mod.rs:35-70) with the trim ranges of
// fov_iterative.rs:59-69, and the temporal filters of zoom_dynamic.rs:15-189 (static and keyframed window).
//
// One CTA per frame: 120 edge points (then <= 4 rounds of 63 interpolated points) are pushed through the inverse lens
// model with their own rolling-shutter rotation in parallel; the order-dependent nearest_edge fold runs on one thread.
// The reference runs this with rayon over frames (fov_iterative.rs:42-56) before rendering starts.
// The rotations are f64, and the slerp's acos / sin differ from glibc's in the last f64 bit, so with the rotation on parity with the
// oracle is to 1e-6.  With suppress_rotation set no libm result reaches the output and the point path is bit-exact.
#include <cuda_runtime.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <thread>
#include <vector>
#include "lens_models.cuh"
#include "warp_kernel.cuh"      // the warp's stage functions: lens correction, refraction, mesh
#include "frame_geometry.cuh"
#include "sync_select.cuh"
#include "gyro_dev.h"
#include "c_abi_internal.h"

using namespace gf;

namespace {

// Everything a point-path kernel reads about one frame: what undistort_points (cpu_undistort.rs:652-698) and at_timestamp_for_points
// (frame_transform.rs:352-438) derive from ComputeParams for it (point_frame).  The lens may change per frame (lens_per_frame), so the
// kernel params and K_new are per frame too.
struct PointFrame {
    gf_kernel_params kp;        // as built by undistort_points (:671-683)
    Track org;                  // device-resident track
    double duration_ms;
    SyncOffsets offsets;        // device-resident multi-point sync offsets (or the scalar)
    double new_k[9];
    int horizontal, suppress_rotation, lens_noop;
    float hstretch, vstretch;   // 0 = do not apply (:702-703)
    float fov, out_cx, out_cy;  // lens-correction blend (:686-694); out_cx 8-byte aligned, so that the kernels load it with out_cy
    Quat q0;                    // smoothed(ts) * org(ts)^-1
    double start_ts, row_readout_time;
    int rs_on;                  // rolling-shutter correction: frame readout time != 0
    CameraStab stab;            // spline points in HBM; absent when at_timestamp_for_points has no shifts (:412, :432-434)
    const double* mesh; uint32_t mesh_len;      // this frame's distorting mesh in HBM (mesh_correction[frame].0), or nullptr
    MeshAux mesh_aux;           // its crop maps and spline steps on the width x height frame
    // the keyframed values at this frame's timestamp (fov_iterative.rs:44-46, frame_transform.rs:354, cpu_undistort.rs:661)
    double rot_c, rot_s;        // video rotation
    float zc_x, zc_y;           // adaptive_zoom_center_offset * input_dim (as f32 products, :100-101)
    float lrc;                  // light refraction coefficient
    int lc; float amount, factor, out_fx, out_fy;       // lens-correction blend (:686-694)
};

// K_new * R for one point — frame_transform.rs:391-410 (f64, no inverted-framebuffer flips), narrowed to f32 like cpu_undistort.rs:764
__device__ void point_rotation(const PointFrame& F, float px, float py, float (&rot)[9]) {
    const double quat_time = F.rs_on ? F.start_ts + F.row_readout_time * (double)(F.horizontal ? px : py) : F.start_ts;
    const Quat q = qmul(F.q0, quat_at_timestamp(F.org, F.duration_ms, F.offsets, quat_time));
    double m[9];
    frame_rotation(q, F.rot_c, F.rot_s, F.new_k, false, F.suppress_rotation, m);
    for (int t = 0; t < 9; ++t) rot[t] = (float)m[t];
}

// The IBIS / OIS shift of point `index` — frame_transform.rs:412-431.  points_iter is the point list when rolling-shutter correction is
// on and the single point (0, 0) otherwise, so with correction off only index 0 has an entry (cpu_undistort.rs:748 `v.get(index)`).
__device__ bool point_shift(const PointFrame& F, float py, size_t index, float (&sh)[5]) {
    if (!F.stab.present) return false;
    if (!F.rs_on && index != 0) return false;
    double s[5];
    stab_shift(F.stab, F.rs_on ? (double)py : 0.0, false, s);
    for (int t = 0; t < 5; ++t) sh[t] = (float)s[t];
    return true;
}

// The mesh block of undistort_points — cpu_undistort.rs:712-746: focal-plane distortion first, then the distorting mesh.  No
// inverted-framebuffer flips on this path.
__device__ void point_mesh(const PointFrame& F, float& x, float& y) {
    const MeshView mesh{ F.mesh };
    const MeshAux& aux = F.mesh_aux;
    const double mesh0 = mesh[0];
    const uint32_t o = as_usize_small(mesh0);
    if (mesh0 > 0.0 && o < F.mesh_len && mesh[o] > 0.0) focal_plane_shift<true>(mesh, aux, o, x, y);     // :714-733 (the reference indexes unchecked)
    if (mesh0 > 10.0) {                                                                                     // :735-745
        x = map_apply(x, aux.to_crop_x);
        y = map_apply(y, aux.to_crop_y);
        const uint32_t n_x = as_usize_small(mesh[1]), n_y = as_usize_small(mesh[2]);
        if (n_x >= 2 && n_x <= GF_MAX_GRID && n_y >= 2 && n_y <= GF_MAX_GRID) {
            double nx, ny;
            mesh_spline(mesh, aux, n_x, n_y, mesh[3], mesh[4], (double)x, (double)y, nx, ny);
            x = (float)nx; y = (float)ny;
        }
        x = map_apply(x, aux.to_frame_x);
        y = map_apply(y, aux.to_frame_y);
    }
}

// one point of undistort_points — cpu_undistort.rs:699-857
template <int LENS, int DIGITAL>
__device__ void undistort_point_rs(const PointFrame& F, float px, float py, size_t index, float& outx, float& outy) {
    const gf_kernel_params& P = F.kp;
    float rot[9];
    point_rotation(F, px, py, rot);                     // rotation time uses the *distorted* point (:393)
    float x = px, y = py;
    if (F.hstretch != 0.0f) x *= F.hstretch;
    if (F.vstretch != 0.0f) y *= F.vstretch;
    if (DIGITAL != GF_LENS_NONE) { float tx, ty; if (Lens<DIGITAL>::undistort(x, y, P, false, tx, ty)) { x = tx; y = ty; } }
    if (F.mesh && F.mesh_len > 9) point_mesh(F, x, y);             // cpu_undistort.rs:712-746
    float sh[5];
    if (point_shift(F, py, index, sh)) {             // cpu_undistort.rs:748-757 (sic: y is rotated with the already rotated x)
        const float cos_a = gf_cosf(sh[2]), sin_a = gf_sinf(sh[2]);
        x = x - P.c[0] - sh[3] + sh[0];
        y = y - P.c[1] - sh[4] + sh[1];
        x = cos_a * x - sin_a * y + P.c[0];
        y = sin_a * x + cos_a * y + P.c[1];
    }
    const float pwx = (x - P.c[0]) / P.f[0], pwy = (y - P.c[1]) / P.f[1];
    float ptx, pty;
    if (!Lens<LENS>::undistort(pwx, pwy, P, F.lens_noop != 0, ptx, pty)) { outx = -1000000.0f; outy = -1000000.0f; return; }
    const bool refract = F.lrc != 1.0f && F.lrc > 0.0f;
    if (refract) refract_undistort(ptx, pty, F.lrc);
    const float pr0 = rot[0] * ptx + rot[1] * pty + rot[2] * 1.0f;
    const float pr1 = rot[3] * ptx + rot[4] * pty + rot[5] * 1.0f;
    const float pr2 = rot[6] * ptx + rot[7] * pty + rot[8] * 1.0f;
    ptx = pr0 / pr2; pty = pr1 / pr2;
    if (F.lc) {                                         // :782-852
        const float amount = F.amount, factor = F.factor, out_fx = F.out_fx, out_fy = F.out_fy;
        const float nx = (ptx - F.out_cx) / out_fx, ny = (pty - F.out_cy) / out_fy;
        float dx, dy;
        Lens<LENS>::distort(nx, ny, 1.0f, P, F.lens_noop != 0, dx, dy);
        float p2x = (dx * out_fx) + F.out_cx, p2y = (dy * out_fy) + F.out_cy;
        if (DIGITAL != GF_LENS_NONE) {
            const float uzx = (p2x - F.out_cx) * F.fov + F.out_cx, uzy = (p2y - F.out_cy) * F.fov + F.out_cy;
            float ddx, ddy;
            Lens<DIGITAL>::distort(uzx, uzy, 1.0f, P, false, ddx, ddy);
            p2x = (ddx - F.out_cx) / F.fov + F.out_cx; p2y = (ddy - F.out_cy) / F.fov + F.out_cy;
        }
        float ox = ptx, oy = pty;
        if (isfinite(p2x) && isfinite(p2y)) { ox = p2x * factor + ptx * amount; oy = p2y * factor + pty * amount; }
        auto r_of = [&](float qx, float qy, float& rx, float& ry) {          // :794-815
            lens_correction_undistort<LENS, DIGITAL>(qx, qy, P, F.out_cx, F.out_cy, out_fx, out_fy, F.fov, F.lens_noop != 0, true, refract, F.lrc, rx, ry);
        };
        for (int it = 0; it < 10; ++it) {
            float rx, ry; r_of(ox, oy, rx, ry);
            const float g0 = amount * ox + factor * rx - ptx, g1 = amount * oy + factor * ry - pty;
            if (fabsf(g0) < 0.02f && fabsf(g1) < 0.02f) break;
            const float eps = 1.0f;
            float rxx, rxy, ryx, ryy;
            r_of(ox + eps, oy, rxx, rxy);
            r_of(ox, oy + eps, ryx, ryy);
            const float j11 = amount + factor * (rxx - rx) / eps, j21 = factor * (rxy - ry) / eps;
            const float j12 = factor * (ryx - rx) / eps,          j22 = amount + factor * (ryy - ry) / eps;
            const float det = j11 * j22 - j12 * j21;
            if (!isfinite(det) || fabsf(det) < 1e-9f) break;
            const float ddx = ( j22 * g0 - j12 * g1) / det, ddy = (-j21 * g0 + j11 * g1) / det;
            if (!isfinite(ddx) || !isfinite(ddy)) break;
            ox = ox - ddx; oy = oy - ddy;
        }
        ptx = ox; pty = oy;
    }
    outx = ptx; outy = pty;
}

constexpr int ZOOM_RECT_LEN = RECT_POINTS;
constexpr int ZOOM_INTERP_LEN = 63;       // (30 + 1) * 3 - 30

// nearest_edge: order-dependent fold over the polygon (fov_iterative.rs:136-151), shrinking (w, h); the index of the last point that
// shrank it, or -1
__device__ int nearest_edge(const float* poly, int plen, float cx, float cy, float inv_aspect, float& w, float& h) {
    int idx = -1;
    for (int i = 0; i < plen; ++i) {
        const float ap0 = fabsf(poly[2 * i] - cx), ap1 = fabsf(poly[2 * i + 1] - cy);
        if (ap0 < w && ap1 < h) {
            if (ap1 > ap0 * inv_aspect) { w = ap1 / inv_aspect; h = ap1; } else { w = ap0; h = ap0 * inv_aspect; }
            idx = i;
        }
    }
    return idx;
}

// The sizes of FovIterative::new (fov_iterative.rs:78-89), the same for every frame of a call
struct FovArgs { float in_w, in_h, out_w, inv_aspect, margin; };

template <int LENS, int DIGITAL>
__global__ void __launch_bounds__(128) find_fov_kernel(const PointFrame* __restrict__ frames, const FovArgs A, double* __restrict__ out) {
    __shared__ float rect[2 * ZOOM_RECT_LEN], poly[2 * ZOOM_RECT_LEN];
    __shared__ float sw, sh; __shared__ int sidx;
    // The frame's record, staged in shared memory: read from global memory instead, the compiler holds more of it in registers across the
    // rounds below (up to 128 per thread instead of 94-126).
    __shared__ PointFrame F;
    const int tid = threadIdx.x;
    for (int i = tid; i < (int)(sizeof(PointFrame) / 8); i += 128) ((unsigned long long*)&F)[i] = ((const unsigned long long*)&frames[blockIdx.x])[i];
    __syncthreads();
    const float cx = A.in_w / 2.0f, cy = A.in_h / 2.0f;
    if (tid < ZOOM_RECT_LEN) {
        float x, y; rect_point(A.in_w, A.in_h, A.margin, tid, x, y);
        rect[2 * tid] = x; rect[2 * tid + 1] = y;
        float ux, uy; undistort_point_rs<LENS, DIGITAL>(F, x, y, (size_t)tid, ux, uy);
        poly[2 * tid] = ux - F.zc_x; poly[2 * tid + 1] = uy - F.zc_y;
    }
    if (tid == 0) { sw = 1000000.0f; sh = 1000000.0f * A.inv_aspect; }
    __syncthreads();
    int plen = ZOOM_RECT_LEN;
    for (int it = 1; it < 5; ++it) {
        if (tid == 0) sidx = nearest_edge(poly, plen, cx, cy, A.inv_aspect, sw, sh);
        __syncthreads();
        const int idx = sidx;
        if (idx < 0) break;
        // relevant = rect[(idx - 1) wrapping % len], rect[idx], rect[(idx + 1) % len]; `idx - 1` wraps through usize::MAX (:117)
        const unsigned long long len = ZOOM_RECT_LEN;
        const int i0 = (int)(((unsigned long long)idx - 1ULL) % len), i1 = idx, i2 = (int)(((unsigned long long)idx + 1ULL) % len);
        float nx = 0.0f, ny = 0.0f;
        if (tid < ZOOM_INTERP_LEN) {                     // interpolate_points(&relevant, 30) :180-189
            const int d = 31, idx1 = tid / d, idx2 = min(idx1 + 1, 2);
            const int ra = idx1 == 0 ? i0 : (idx1 == 1 ? i1 : i2), rb = idx2 == 1 ? i1 : i2;
            const float f = (float)(tid % d) / (float)d;
            const float dx = rect[2 * ra] + f * (rect[2 * rb] - rect[2 * ra]);
            const float dy = rect[2 * ra + 1] + f * (rect[2 * rb + 1] - rect[2 * ra + 1]);
            undistort_point_rs<LENS, DIGITAL>(F, dx, dy, (size_t)tid, nx, ny);
        }
        __syncthreads();                                 // everyone has read rect/poly of this round
        if (tid < ZOOM_INTERP_LEN) { poly[2 * tid] = nx - F.zc_x; poly[2 * tid + 1] = ny - F.zc_y; }
        plen = ZOOM_INTERP_LEN;
        __syncthreads();
        if (tid == 0) (void)nearest_edge(poly, plen, cx, cy, A.inv_aspect, sw, sh);       // :127 nearest_edge again (index discarded)
        __syncthreads();
    }
    if (tid == 0) out[blockIdx.x] = (double)(sw * 2.0f / A.out_w);      // :133
}

// undistort_points over an explicit point list (pts != nullptr: out = n x (x, y)) or over every pixel centre of a w x h grid
// (pts == nullptr: out = w*h x RGB, the ST-map encoding of stmap.rs:131-135: x / w, 1 - y / h, 0).
template <int LENS, int DIGITAL>
__global__ void __launch_bounds__(128) points_kernel(const __grid_constant__ PointFrame F, const float2* __restrict__ pts, size_t n, int grid_w, int grid_h, float* __restrict__ out) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float px, py;
    if (pts) { const float2 p = pts[i]; px = p.x; py = p.y; }
    else     { px = (float)(int)(i % (size_t)grid_w); py = (float)(int)(i / (size_t)grid_w); }
    float ox, oy;
    undistort_point_rs<LENS, DIGITAL>(F, px, py, pts ? i : (size_t)0, ox, oy);      // ST map: every pixel is its own one-point call (stmap.rs:114-116)
    if (pts) { out[2 * i] = ox; out[2 * i + 1] = oy; }
    else     { out[3 * i] = ox / (float)grid_w; out[3 * i + 1] = 1.0f - (oy / (float)grid_h); out[3 * i + 2] = 0.0f; }
}
// The undistorted size of one frame per CTA — stmap.rs:58-77: the 120 points_around_rect(w, h, 31, 31) edge points with margin 0
// (fov_iterative.rs:154-175) through undistort_points, their bounding box folded in order from 0 with f32::min / max (NaN is
// ignored, :62-71), then `ceil(max - min) as usize` for each extent.
template <int LENS, int DIGITAL>
__global__ void __launch_bounds__(128) stmap_size_kernel(const PointFrame* __restrict__ frames, float w, float h, int2* __restrict__ out) {
    __shared__ float und[2 * RECT_POINTS];
    const PointFrame& F = frames[blockIdx.x];
    const int tid = threadIdx.x;
    if (tid < RECT_POINTS) {
        float x, y; rect_point(w, h, 0.0f, tid, x, y);
        undistort_point_rs<LENS, DIGITAL>(F, x, y, (size_t)tid, und[2 * tid], und[2 * tid + 1]);
    }
    __syncthreads();
    if (tid != 0) return;
    float min_x = 0.0f, min_y = 0.0f, max_x = 0.0f, max_y = 0.0f;
    for (int i = 0; i < RECT_POINTS; ++i) {
        min_x = fminf(und[2 * i], min_x); min_y = fminf(und[2 * i + 1], min_y);
        max_x = fmaxf(und[2 * i], max_x); max_y = fmaxf(und[2 * i + 1], max_y);
    }
    const float fw = ceilf(max_x - min_x), fh = ceilf(max_y - min_y);
    // `as usize`: truncating, saturating, NaN -> 0 (kept within int32; anything that large is out of range anyway)
    auto as_size = [](float v) { return v != v ? 0 : (v <= 0.0f ? 0 : (v >= 2147483647.0f ? 2147483647 : (int)v)); };
    out[blockIdx.x] = make_int2(as_size(fw), as_size(fh));
}

// ---- visual-features sync: calculate_distance (synchronization/find_offset/visual_features.rs:46-84) ----
struct SyncPairDev { uint32_t off, n; };        // a pair's first point in the concatenated lists, and its point count

// One CTA per (candidate, pair).  recs: 2 records per CTA (the pair's two timestamps at this candidate), blockIdx.x = candidate *
// n_pairs + pair.  Every thread undistorts its points, keeps the truncated f32 squared distance of each point pair inside the frame as a
// 32-bit key, and sync_select_add (sync_select.cuh) adds the sum of the k smallest keys to sums[candidate].
template <int LENS, int DIGITAL>
__global__ void __launch_bounds__(SYNC_THREADS) sync_cost_kernel(const PointFrame* __restrict__ recs, const SyncPairDev* __restrict__ pairs, unsigned n_pairs,
                                                                 const float2* __restrict__ pts1, const float2* __restrict__ pts2, float w, float h,
                                                                 uint32_t* __restrict__ scratch, size_t scratch_stride, unsigned long long* __restrict__ sums) {
    extern __shared__ uint32_t skeys[];
    __shared__ unsigned hist[256];
    __shared__ uint64_t red[SYNC_THREADS / 32];
    __shared__ uint32_t s_prefix, s_rank;
    const unsigned cand = blockIdx.x / n_pairs;
    const SyncPairDev pr = pairs[blockIdx.x % n_pairs];
    if (pr.n == 0) return;
    uint32_t* keys = pr.n <= SYNC_SMEM_KEYS ? skeys : scratch + (size_t)cand * scratch_stride + pr.off;
    const PointFrame& S1 = recs[2 * (size_t)blockIdx.x];
    const PointFrame& S2 = recs[2 * (size_t)blockIdx.x + 1];
    uint64_t valid = 0;
    for (uint32_t i = threadIdx.x; i < pr.n; i += SYNC_THREADS) {
        const float2 a = pts1[pr.off + i], b = pts2[pr.off + i];
        float x1, y1, x2, y2;
        undistort_point_rs<LENS, DIGITAL>(S1, a.x, a.y, (size_t)i, x1, y1);
        undistort_point_rs<LENS, DIGITAL>(S2, b.x, b.y, (size_t)i, x2, y2);
        uint32_t key = SYNC_NO_KEY;
        if (x1 > 0.0f && x1 < w && y1 > 0.0f && y1 < h && x2 > 0.0f && x2 < w && y2 > 0.0f && y2 < h) {      // :66-67
            const float dx = x2 - x1, dy = y2 - y1;
            key = (uint32_t)(dx * dx + dy * dy);         // `dist as u64` (no contraction: built with -fmad=false)
            ++valid;
        }
        keys[i] = key;
    }
    sync_select_add(keys, pr.n, valid, hist, red, s_prefix, s_rank, &sums[cand]);
}

// The kernels of a (lens, digital lens) pair, compiled only for the pairs the reference combines (the GoPro views need the fisheye
// model, GoPro warp the GoPro model); nullptr for any other pair.
struct ZoomKernels {
    void (*find_fov)(const PointFrame*, const FovArgs, double*);
    void (*points)(const PointFrame, const float2*, size_t, int, int, float*);
    void (*stmap_size)(const PointFrame*, float, float, int2*);
    void (*sync_cost)(const PointFrame*, const SyncPairDev*, unsigned, const float2*, const float2*, float, float, uint32_t*, size_t, unsigned long long*);
};
template <int LENS, int DIGITAL> const ZoomKernels* kernels_of() {
    static const ZoomKernels k{ find_fov_kernel<LENS, DIGITAL>, points_kernel<LENS, DIGITAL>, stmap_size_kernel<LENS, DIGITAL>, sync_cost_kernel<LENS, DIGITAL> };
    return &k;
}
template <int LENS> const ZoomKernels* pick_digital(int digital) {
    switch (digital) {
    case GF_LENS_NONE:             return kernels_of<LENS, GF_LENS_NONE>();
    case GF_LENS_DIGITAL_STRETCH:  return kernels_of<LENS, GF_LENS_DIGITAL_STRETCH>();
    case GF_LENS_GOPRO_SUPERVIEW:  if constexpr (LENS == GF_LENS_OPENCV_FISHEYE) return kernels_of<LENS, GF_LENS_GOPRO_SUPERVIEW>();  break;
    case GF_LENS_GOPRO6_SUPERVIEW: if constexpr (LENS == GF_LENS_OPENCV_FISHEYE) return kernels_of<LENS, GF_LENS_GOPRO6_SUPERVIEW>(); break;
    case GF_LENS_GOPRO_HYPERVIEW:  if constexpr (LENS == GF_LENS_OPENCV_FISHEYE) return kernels_of<LENS, GF_LENS_GOPRO_HYPERVIEW>();  break;
    case GF_LENS_GOPRO_WARP:       if constexpr (LENS == GF_LENS_GOPRO) return kernels_of<LENS, GF_LENS_GOPRO_WARP>();                break;
    default: break;
    }
    return nullptr;
}
const ZoomKernels* pick_kernels(int lens, int digital) {
    switch (lens) {
    case GF_LENS_OPENCV_FISHEYE:     return pick_digital<GF_LENS_OPENCV_FISHEYE>(digital);
    case GF_LENS_OPENCV_STANDARD:    return pick_digital<GF_LENS_OPENCV_STANDARD>(digital);
    case GF_LENS_POLY3:              return pick_digital<GF_LENS_POLY3>(digital);
    case GF_LENS_POLY5:              return pick_digital<GF_LENS_POLY5>(digital);
    case GF_LENS_PTLENS:             return pick_digital<GF_LENS_PTLENS>(digital);
    case GF_LENS_INSTA360:           return pick_digital<GF_LENS_INSTA360>(digital);
    case GF_LENS_SONY:               return pick_digital<GF_LENS_SONY>(digital);
    case GF_LENS_GENERIC_POLYNOMIAL: return pick_digital<GF_LENS_GENERIC_POLYNOMIAL>(digital);
    case GF_LENS_GOPRO:              return pick_digital<GF_LENS_GOPRO>(digital);
    default: return nullptr;
    }
}

} // namespace

// at_timestamp_for_points' fov without focal-length compensation (frame_transform.rs:360-362): get_fov, scaled by the output size as
// (fov * width) / output_width
static double points_fov(const gf_compute_params* cp, size_t frame, bool use_fovs, double timestamp_ms) {
    return fov_unscaled(cp, frame, use_fovs, timestamp_ms, false) * (double)cp->width / (double)(cp->output_width > 1 ? cp->output_width : 1);
}

// What the callers of point_frame choose, in this order
struct PointOpts {
    bool use_fovs = false;                  // get_fov with the clip's fovs
    double lens_correction_amount = 1.0;    // the lens-correction strength
    bool zoom_keys = false;                 // find_fov (fov_iterative.rs:44-46): the zoom centre and the strength follow their tracks,
                                            // lens_correction_amount being the strength without one
    bool clear_offsets = false;             // the offset search (visual_features.rs:14 clear_offsets): no gyro or sync offsets, on the host
                                            // or the device
};
// One frame of undistort_points at timestamp `ts`.  The lens is get_lens_data_at_timestamp of this frame (frame_transform.rs:360) for ONE
// timestamp: the per-frame lens in a private copy of `cp_user`.  From it: kernel params and K_new, readout timing, smoothed(ts) *
// org(ts)^-1, shifts and distorting mesh (frame_transform.rs:366-388, 412-434), video rotation (:354), refraction (cpu_undistort.rs:661)
// and the lens-correction blend (:686-694).
static PointFrame point_frame(const gf_cuda_gyro* g, const gf_compute_params& cp_user, int distortion_model, size_t frame, double ts,
                              const PointOpts& o) {
    gf_compute_params cp = cp_user;
    if (cp_user.lens_per_frame && frame < cp_user.n_lens_per_frame) {
        const gf_lens_data& L = cp_user.lens_per_frame[frame];
        memcpy(cp.camera_matrix, L.camera_matrix, sizeof(cp.camera_matrix)); memcpy(cp.distortion_coeffs, L.distortion_coeffs, sizeof(cp.distortion_coeffs));
        cp.radial_distortion_limit = L.radial_distortion_limit;
    }
    if (o.clear_offsets) { cp.gyro_offset_ms = 0.0; cp.sync_offset_ts_us = nullptr; cp.sync_offset_ms = nullptr; cp.n_sync_offsets = 0; }
    PointFrame f{};
    const double fov = points_fov(&cp, frame, o.use_fovs, ts);
    const double* K = cp.camera_matrix;
    get_new_k(&cp, K, fov, f.new_k);
    f.horizontal = cp.readout_horizontal; f.suppress_rotation = cp.suppress_rotation;
    f.org = g->org_track();
    f.duration_ms = cp.duration_ms;
    f.offsets = o.clear_offsets ? SyncOffsets{} : g->sync_offsets(cp.gyro_offset_ms);
    gf_kernel_params& kp = f.kp;                                                            // cpu_undistort.rs:671-683
    kp.width = cp.width; kp.height = cp.height; kp.output_width = cp.output_width; kp.output_height = cp.output_height;
    kp.f[0] = (float)K[0]; kp.f[1] = (float)K[4]; kp.c[0] = (float)K[2]; kp.c[1] = (float)K[5];
    for (int i = 0; i < 12; ++i) kp.k[i] = (float)cp.distortion_coeffs[i];
    for (int i = 0; i < 16 && i < cp.n_digital_lens_params; ++i) kp.digital_lens_params[i] = (float)cp.digital_lens_params[i];
    f.lens_noop = lens_noop(distortion_model, kp.k) ? 1 : 0;
    f.hstretch = cp.input_horizontal_stretch > 0.001 ? (float)cp.input_horizontal_stretch : 0.0f;
    f.vstretch = cp.input_vertical_stretch   > 0.001 ? (float)cp.input_vertical_stretch   : 0.0f;
    f.out_cx = (float)cp.output_width / 2.0f; f.out_cy = (float)cp.output_height / 2.0f; f.fov = (float)fov;

    const FrameTiming t = frame_timing(&cp, frame, ts, false);
    f.q0 = t.q0; f.start_ts = t.start_ts; f.row_readout_time = t.row_readout_time;
    f.rs_on = fabs(t.frame_readout_time) > 0.0 ? 1 : 0;
    f.mesh = g->frame_mesh(frame, f.mesh_len);
    if (f.mesh) make_mesh_aux(g->mesh_index[frame].header, (float)cp.width, (float)cp.height, f.mesh_aux);
    StabSplines sp;
    const bool shifts = !(cp.suppress_rotation && cp.frame_readout_time == 0.0) && g->frame_splines(frame, sp);       // :432-434
    f.stab = camera_stab_at(&cp, frame, false, shifts ? &sp : nullptr);
    const double a = keyframed(&cp, GF_KF_VIDEO_ROTATION, ts, cp.video_rotation) * (M_PI / 180.0);
    f.rot_c = cos(a); f.rot_s = sin(a);
    f.lrc = (float)keyframed(&cp, GF_KF_LIGHT_REFRACTION_COEFF, ts, cp.light_refraction_coefficient);
    double lca = o.lens_correction_amount;
    if (o.zoom_keys) {
        f.zc_x = (float)keyframed(&cp, GF_KF_ZOOMING_CENTER_X, ts, cp.adaptive_zoom_center_offset[0]) * (float)cp.width;
        f.zc_y = (float)keyframed(&cp, GF_KF_ZOOMING_CENTER_Y, ts, cp.adaptive_zoom_center_offset[1]) * (float)cp.height;
        lca = keyframed(&cp, GF_KF_LENS_CORRECTION_STRENGTH, ts, o.lens_correction_amount);
    }
    f.lc = lca < 1.0 ? 1 : 0;
    f.amount = (float)lca; f.factor = fmaxf(1.0f - f.amount, 0.001f);
    f.out_fx = kp.f[0] / f.fov / f.factor; f.out_fy = kp.f[1] / f.fov / f.factor;
    return f;
}

bool gf::point_path_supported(int lens, int digital) { return pick_kernels(lens, digital) != nullptr; }

// The synchronous calls: `in` to a device buffer of the call, launch(d_in, d_out, stream), `out` back from one, then wait for the stream.
template <class In, class Out, class Launch>
static int round_trip(gf_cuda_gyro* g, void* cu_stream, const In* in, size_t n_in, Out* out, size_t n_out, Launch launch) {
    const cudaStream_t st = g->stream_of(cu_stream);
    GrowBuf<In> d_in; GrowBuf<Out> d_out;
    CK(nullptr, d_in.reserve(n_in, st));
    CK(nullptr, d_out.reserve(n_out, st));
    CK(nullptr, cudaMemcpyAsync(d_in.ptr, in, n_in * sizeof(In), cudaMemcpyHostToDevice, st));
    launch(d_in.ptr, d_out.ptr, st);
    CK(nullptr, cudaGetLastError());
    CK(nullptr, cudaMemcpyAsync(out, d_out.ptr, n_out * sizeof(Out), cudaMemcpyDeviceToHost, st));
    CK(nullptr, cudaStreamSynchronize(st));
    return GF_OK;
}

// ---- visual-features sync on the host: argument checks, point records in chunks of candidates, the two-stage search ----

// frame_at_timestamp (lib.rs:2069): `(timestamp_ms * (fps / 1000.0)).round() as i32`, then `as usize`, so a negative frame wraps
static size_t sync_frame(double timestamp_ms, double fps) {
    const double r = round(timestamp_ms * (fps / 1000.0));
    const int32_t i = r != r ? 0 : (r <= -2147483648.0 ? INT32_MIN : (r >= 2147483647.0 ? INT32_MAX : (int32_t)r));
    return (size_t)(int64_t)i;
}

constexpr size_t kSyncChunkBytes = 64u << 20;          // records (and global key scratch) of one chunk of candidates
constexpr double kMaxSyncCandidates = 1e7;             // per search stage

// The pairs of one range on the device, and what every cost evaluation over them shares.
struct SyncJob {
    gf_cuda_gyro* g; const gf_compute_params* cp; int model; double fps; int clear;
    const gf_sync_pair* pairs; size_t n_pairs;
    const ZoomKernels* k; cudaStream_t st;
    size_t total = 0; uint32_t max_n = 0;
    GrowBuf<float2> d_p1, d_p2; GrowBuf<SyncPairDev> d_pairs; GrowBuf<PointFrame> d_recs; GrowBuf<uint32_t> d_scratch;
    GrowBuf<unsigned long long> d_sums;
};

// Everything the cost calls refuse, before any CUDA call: GF_OK or the error, with `who` in the message.
static int sync_check(const char* who, const gf_cuda_gyro* g, const gf_compute_params* cp, int model, int digital, double fps,
                      const gf_sync_pair* pairs, size_t n_pairs) {
    const std::string w(who);
    if (!g || !cp || (n_pairs && !pairs)) return fail(nullptr, GF_ERR_BAD_PARAMS, w + ": null argument");
    if (!pick_kernels(model, digital)) return fail(nullptr, GF_ERR_UNSUPPORTED_COMBO, w + ": no point-path kernel for this (lens, digital lens) pair");
    if (cp->width < 1 || cp->height < 1 || cp->width > 32768 || cp->height > 32768)
        return fail(nullptr, GF_ERR_BAD_PARAMS, w + ": frame size outside 1..32768");
    if (!(fps > 0.0) || !std::isfinite(fps)) return fail(nullptr, GF_ERR_BAD_PARAMS, w + ": scaled_fps must be finite and > 0");
    unsigned __int128 total = 0;
    for (size_t p = 0; p < n_pairs; ++p) {
        if (pairs[p].n && (!pairs[p].pts1 || !pairs[p].pts2)) return fail(nullptr, GF_ERR_BAD_PARAMS, w + ": pair " + std::to_string(p) + " has a null point list");
        total += pairs[p].n;
    }
    if (total > 0xFFFFFFFFu) return fail(nullptr, GF_ERR_BAD_PARAMS, w + ": more than 2^32 - 1 points");
    // every distance is below width^2 + height^2, so below this bound the f64 sum of the reference is exact and equals the integer sum
    const unsigned __int128 d2 = (unsigned __int128)cp->width * cp->width + (unsigned __int128)cp->height * cp->height;
    if (total * d2 >= ((unsigned __int128)1 << 53))
        return fail(nullptr, GF_ERR_BAD_PARAMS, w + ": sum(n) * (width^2 + height^2) reaches 2^53, the cost would not be exact in f64");
    return GF_OK;
}

static int sync_setup(SyncJob& J) {
    std::vector<float2> h1, h2; std::vector<SyncPairDev> hp(J.n_pairs);
    for (size_t p = 0; p < J.n_pairs; ++p) {
        const gf_sync_pair& P = J.pairs[p];
        hp[p] = SyncPairDev{ (uint32_t)h1.size(), (uint32_t)P.n };
        J.max_n = std::max(J.max_n, (uint32_t)P.n);
        for (size_t i = 0; i < P.n; ++i) { h1.push_back(make_float2(P.pts1[2 * i], P.pts1[2 * i + 1])); h2.push_back(make_float2(P.pts2[2 * i], P.pts2[2 * i + 1])); }
    }
    J.total = h1.size();
    if (J.total == 0) return GF_OK;
    CK(nullptr, J.d_p1.reserve(J.total, J.st));
    CK(nullptr, J.d_p2.reserve(J.total, J.st));
    CK(nullptr, J.d_pairs.reserve(J.n_pairs, J.st));
    CK(nullptr, cudaMemcpyAsync(J.d_p1.ptr, h1.data(), J.total * sizeof(float2), cudaMemcpyHostToDevice, J.st));
    CK(nullptr, cudaMemcpyAsync(J.d_p2.ptr, h2.data(), J.total * sizeof(float2), cudaMemcpyHostToDevice, J.st));
    CK(nullptr, cudaMemcpyAsync(J.d_pairs.ptr, hp.data(), J.n_pairs * sizeof(SyncPairDev), cudaMemcpyHostToDevice, J.st));
    CK(nullptr, cudaStreamSynchronize(J.st));           // the staging vectors go out of scope
    return GF_OK;
}

// The records of candidates c0 .. c0 + nc: per pair, what gf_cuda_undistort_points builds for each of its two timestamps, on all host
// threads (point_frame only reads).
static void sync_records(const SyncJob& J, const double* offs, const double* rs, size_t c0, size_t nc, PointFrame* out) {
    auto work = [&](size_t a, size_t b) {
        gf_compute_params cp = *J.cp;
        const PointOpts o{ false, 1.0, false, J.clear != 0 };
        for (size_t c = a; c < b; ++c) {
            const double off = offs ? offs[c0 + c] : 0.0;
            if (rs) cp.frame_readout_time = rs[c0 + c];
            for (size_t p = 0; p < J.n_pairs; ++p) {
                const gf_sync_pair& P = J.pairs[p];
                const double t1 = (double)P.ts_us / 1000.0 - off, t2 = (double)P.next_ts_us / 1000.0 - off;     // :60-64
                PointFrame* r = out + 2 * (c * J.n_pairs + p);
                r[0] = point_frame(J.g, cp, J.model, sync_frame(t1, J.fps), t1, o);
                r[1] = point_frame(J.g, cp, J.model, sync_frame(t2, J.fps), t2, o);
            }
        }
    };
    const size_t nt = std::min<size_t>({ (size_t)std::max(1u, std::thread::hardware_concurrency()), 16, (nc * J.n_pairs + 63) / 64, nc });
    if (nt <= 1) { work(0, nc); return; }
    std::vector<std::thread> th;
    for (size_t t = 0; t < nt; ++t) th.emplace_back(work, nc * t / nt, nc * (t + 1) / nt);
    for (auto& t : th) t.join();
}

// calculate_distance of n candidates over the job's pairs into out[]
static int sync_run(SyncJob& J, const double* offs, const double* rs, size_t n, double* out) {
    if (n == 0) return GF_OK;
    if (J.total == 0) { for (size_t c = 0; c < n; ++c) out[c] = 0.0; return GF_OK; }
    const bool big = J.max_n > SYNC_SMEM_KEYS;
    const size_t per_cand = 2 * J.n_pairs * sizeof(PointFrame) + (big ? J.total * sizeof(uint32_t) : 0);
    const size_t chunk = std::min({ std::max<size_t>(1, kSyncChunkBytes / per_cand), n, (size_t)0x7fffffff / J.n_pairs });
    std::vector<PointFrame> host(2 * chunk * J.n_pairs);
    CK(nullptr, J.d_recs.reserve(host.size(), J.st));
    if (big) CK(nullptr, J.d_scratch.reserve(chunk * J.total, J.st));
    CK(nullptr, J.d_sums.reserve(n, J.st));
    CK(nullptr, cudaMemsetAsync(J.d_sums.ptr, 0, n * sizeof(unsigned long long), J.st));
    cudaEvent_t e[2] = {};
    CK(nullptr, cudaEventCreate(&e[0]));
    const Event ev0(e[0]);
    CK(nullptr, cudaEventCreate(&e[1]));
    const Event ev1(e[1]);
    const unsigned smem = std::min<unsigned>(J.max_n, SYNC_SMEM_KEYS) * (unsigned)sizeof(uint32_t);
    float ms = 0.0f;
    for (size_t c0 = 0; c0 < n; c0 += chunk) {
        const size_t nc = std::min(chunk, n - c0);
        const auto t0 = std::chrono::steady_clock::now();
        sync_records(J, offs, rs, c0, nc, host.data());
        J.g->sync_host_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (c0) { CK(nullptr, cudaEventSynchronize(e[1])); CK(nullptr, cudaEventElapsedTime(&ms, e[0], e[1])); J.g->sync_device_ms += ms; }
        // pageable source: the call returns once the records are staged, so the next chunk may overwrite `host`
        CK(nullptr, cudaMemcpyAsync(J.d_recs.ptr, host.data(), 2 * nc * J.n_pairs * sizeof(PointFrame), cudaMemcpyHostToDevice, J.st));
        CK(nullptr, cudaEventRecord(e[0], J.st));
        J.k->sync_cost<<<(unsigned)(nc * J.n_pairs), SYNC_THREADS, smem, J.st>>>(J.d_recs.ptr, J.d_pairs.ptr, (unsigned)J.n_pairs, J.d_p1.ptr, J.d_p2.ptr,
                                                                               (float)J.cp->width, (float)J.cp->height, big ? J.d_scratch.ptr : nullptr,
                                                                               J.total, J.d_sums.ptr + c0);
        CK(nullptr, cudaGetLastError());
        CK(nullptr, cudaEventRecord(e[1], J.st));
        ++J.g->sync_chunks;
    }
    std::vector<unsigned long long> sums(n);
    CK(nullptr, cudaMemcpyAsync(sums.data(), J.d_sums.ptr, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, J.st));
    CK(nullptr, cudaStreamSynchronize(J.st));
    CK(nullptr, cudaEventElapsedTime(&ms, e[0], e[1])); J.g->sync_device_ms += ms;
    for (size_t c = 0; c < n; ++c) out[c] = (double)sums[c];        // exact: every sum is below 2^53 (sync_check)
    return GF_OK;
}

// find_min under reduce_with (:87): `if a.1 < b.1 { a } else { b }` folded in order keeps the LAST of equal minima
static size_t sync_last_min(const std::vector<double>& cost) {
    size_t b = 0;
    for (size_t i = 1; i < cost.size(); ++i) if (!(cost[b] < cost[i])) b = i;
    return b;
}

// ---- the temporal filters of zoom_dynamic.rs, on the host like in the reference ----

// Rust's `f64 as usize`: truncates, saturates, NaN -> 0
static size_t as_usize(double x) {
    if (!(x > 0.0)) return 0;
    return x >= 18446744073709551616.0 ? SIZE_MAX : (size_t)x;
}
// KeyframeManager::is_keyframed for a flattened track (the custom provider is baked into the track by the caller)
static bool track_keyed(const gf_keyframe_track& t) { return t.n > 0 && t.ts_us && t.value; }

// envelope_follower (zoom_dynamic.rs:165-189): alphas[i] belongs to sample i in both passes
static std::vector<double> envelope_follower(const std::vector<double>& a, const std::vector<double>& alphas) {
    const size_t m = a.size(); std::vector<double> rev(m), res(m);
    double q = a[m - 1];
    for (size_t r = 0; r < m; ++r) { const size_t i = m - 1 - r; const double x = a[i], al = alphas[i]; q = fmin(x, x * al + q * (1.0 - al)); rev[r] = q; }
    q = rev[m - 1];
    for (size_t r = 0; r < m; ++r) { const double x = rev[m - 1 - r], al = alphas[r]; q = fmin(x, x * al + q * (1.0 - al)); res[r] = q; }
    return res;
}

// Windows longer than this many frames are rejected instead of allocated (the reference would panic on the allocation).
constexpr double kMaxWindowFrames = 1e8;

// zoom_dynamic::compute's static-window branch (zoom_dynamic.rs:56-76) in place on v (non-empty).  False when the window is too long.
static bool zoom_static_window(std::vector<double>& v, double window_s, double fps, int method) {
    const size_t n = v.size();
    if (method == 1) {
        v = envelope_follower(v, std::vector<double>(n, 1.0 - exp(-(1.0 / fps) / window_s)));
        v = envelope_follower(v, std::vector<double>(n, 1.0 - exp(-(1.0 / fps) / 0.2)));
        return true;
    }
    const double frames_f = floor(window_s * fps);                  // get_frames_per_window :82-88
    if (frames_f >= kMaxWindowFrames) return false;
    size_t frames = as_usize(frames_f); if (frames % 2 == 0) frames += 1;
    const size_t half = frames / 2;
    auto pad = [&](const std::vector<double>& a) { std::vector<double> p(a.size() + 2 * half); for (size_t i = 0; i < p.size(); ++i) p[i] = i < half ? a.front() : (i >= half + a.size() ? a.back() : a[i - half]); return p; };
    std::vector<double> p = pad(v), mn(n);
    for (size_t i = 0; i < n; ++i) { double m = p[i]; for (size_t j = 1; j < frames; ++j) m = fmin(m, p[i + j]); mn[i] = m; }
    p = pad(mn);
    std::vector<double> gw(frames); const double sd = (double)frames / 6.0, sig2 = 2.0 * sd * sd; double sum = 0.0;
    for (size_t i = 0; i < frames; ++i) { const long x = (long)i - (long)half; gw[i] = exp(-(double)(x * x) / sig2); sum += gw[i]; }
    for (auto& w : gw) w /= sum;
    for (size_t i = 0; i < n; ++i) { double s = 0.0; for (size_t j = 0; j < frames; ++j) s += p[i + j] * gw[j]; v[i] = s; }
    return true;
}


extern "C" {

// FovIterative::compute for `n` frames (zooming/fov_iterative.rs:31-74 without trim ranges): out[i] = find_fov(frame i), with the frame's
// keyframed zoom centre / lens-correction strength (:41-52), video rotation and refraction when gf_compute_params carries those tracks.
// `cp` is the user's ComputeParams; the calculate_fovs adjustments (fov_scale = 1, fovs cleared, output size = input size,
// zooming/mod.rs:41-49) are applied here.
GF_API int gf_cuda_find_fovs(gf_cuda_gyro* g, const gf_compute_params* cp_user, int distortion_model, int digital_lens,
                             const double* timestamps_ms, size_t n, float fov_algorithm_margin, double* out_fov_minimal, void* cu_stream) {
    if (!g || !cp_user || !timestamps_ms || !out_fov_minimal) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_find_fovs: null argument");
    if (n == 0) return GF_OK;
    const ZoomKernels* k = pick_kernels(distortion_model, digital_lens);
    if (!k) return fail(nullptr, GF_ERR_UNSUPPORTED_COMBO, "gf_cuda_find_fovs: no point-path kernel for this (lens, digital lens) pair");
    CK(nullptr, cudaSetDevice(g->device));
    gf_compute_params cp = *cp_user;
    const int org_ow = cp.output_width, org_oh = cp.output_height;
    cp.fov_scale = 1.0; cp.n_fovs = 0; cp.n_minimal_fovs = 0; cp.output_width = cp.width; cp.output_height = cp.height;
    cp.lens_per_frame = nullptr; cp.n_lens_per_frame = 0;          // the FOVs are those of the clip's base lens

    FovArgs A;
    const float ratio = (float)cp.width / (float)(org_ow > 1 ? org_ow : 1);                // FovIterative::new :78-89
    A.in_w = (float)cp.width; A.in_h = (float)cp.height;
    A.out_w = (float)org_ow * ratio; const float out_h = (float)org_oh * ratio;
    A.inv_aspect = out_h / A.out_w; A.margin = fov_algorithm_margin;
    // use_fovs = false: every record's fov is 1 after the adjustments
    const PointOpts o{ false, cp.lens_correction_amount, true };
    std::vector<PointFrame> hf(n);
    for (size_t i = 0; i < n; ++i) hf[i] = point_frame(g, cp, distortion_model, i, timestamps_ms[i], o);
    return round_trip(g, cu_stream, hf.data(), n, out_fov_minimal, n, [&](const PointFrame* d_in, double* d_out, cudaStream_t st) {
        k->find_fov<<<(unsigned)n, 128, 0, st>>>(d_in, A, d_out);
    });
}

// undistort_points_with_rolling_shutter for an arbitrary point list (cpu_undistort.rs:636-641): host in / host out, synchronous.
GF_API int gf_cuda_undistort_points(gf_cuda_gyro* g, const gf_compute_params* cp_user, int distortion_model, int digital_lens,
                                    double timestamp_ms, size_t frame, int use_fovs, double lens_correction_amount,
                                    const float* points_xy, size_t n, float* out_xy, void* cu_stream) {
    if (!g || !cp_user || !points_xy || !out_xy) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_undistort_points: null argument");
    if (n == 0) return GF_OK;
    const ZoomKernels* k = pick_kernels(distortion_model, digital_lens);
    if (!k) return fail(nullptr, GF_ERR_UNSUPPORTED_COMBO, "gf_cuda_undistort_points: no point-path kernel for this (lens, digital lens) pair");
    CK(nullptr, cudaSetDevice(g->device));
    const PointFrame p = point_frame(g, *cp_user, distortion_model, frame, timestamp_ms, PointOpts{ use_fovs != 0, lens_correction_amount });
    return round_trip(g, cu_stream, (const float2*)points_xy, n, out_xy, n * 2, [&](const float2* d_in, float* d_out, cudaStream_t st) {
        k->points<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(p, d_in, n, 0, 0, d_out);
    });
}

// The "redistort" ST map (stmap.rs:112-116): undistort_points of every pixel centre of the width x height frame, written to
// device memory as RGB f32 (x / width, 1 - y / height, 0).  Asynchronous on the stream.
GF_API int gf_cuda_stmap_distort_dev(gf_cuda_gyro* g, const gf_compute_params* cp_user, int distortion_model, int digital_lens,
                                     double timestamp_ms, size_t frame, float* out_rgb_dev, void* cu_stream) {
    if (!g || !cp_user || !out_rgb_dev) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_stmap_distort_dev: null argument");
    const ZoomKernels* k = pick_kernels(distortion_model, digital_lens);
    if (!k) return fail(nullptr, GF_ERR_UNSUPPORTED_COMBO, "gf_cuda_stmap_distort_dev: no point-path kernel for this (lens, digital lens) pair");
    const int w = cp_user->width, h = cp_user->height;
    if (w < 1 || h < 1) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_stmap_distort_dev: frame size < 1");
    CK(nullptr, cudaSetDevice(g->device));
    const PointFrame p = point_frame(g, *cp_user, distortion_model, frame, timestamp_ms, PointOpts{ true });
    const size_t n = (size_t)w * (size_t)h;
    k->points<<<(unsigned)((n + 127) / 128), 128, 0, g->stream_of(cu_stream)>>>(p, nullptr, n, w, h, out_rgb_dev);
    CK(nullptr, cudaGetLastError());
    return GF_OK;
}

// The undistorted size of every frame of an ST-map job (stmap.rs:58-77), one CTA per frame.  Each frame's record is what
// gf_cuda_undistort_points(use_fovs = 0, lens_correction_amount = 1) builds for it, so the sizes are those of gf_cuda_generate_stmap.
GF_API int gf_cuda_stmap_sizes(gf_cuda_gyro* g, const gf_compute_params* cp_user, int distortion_model, int digital_lens, int per_frame,
                               const size_t* frames, const double* timestamps_ms, size_t n,
                               int32_t* out_new_width, int32_t* out_new_height, void* cu_stream) {
    if (!g || !cp_user) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_stmap_sizes: null argument");
    if (n == 0) return GF_OK;
    if (!frames || !timestamps_ms || !out_new_width || !out_new_height) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_stmap_sizes: null argument");
    if (n > 0x7fffffffu) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_stmap_sizes: too many frames");
    const gf_compute_params cp = stmap_params(*cp_user, per_frame);
    if (cp.width < 4 || cp.height < 4) return fail(nullptr, GF_ERR_SIZE_TOO_SMALL, "gf_cuda_stmap_sizes: SizeTooSmall");
    const ZoomKernels* k = pick_kernels(distortion_model, digital_lens);
    if (!k) return fail(nullptr, GF_ERR_UNSUPPORTED_COMBO, "gf_cuda_stmap_sizes: no point-path kernel for this (lens, digital lens) pair");
    CK(nullptr, cudaSetDevice(g->device));
    std::vector<PointFrame> hf(n);
    for (size_t i = 0; i < n; ++i) hf[i] = point_frame(g, cp, distortion_model, frames[i], timestamps_ms[i], PointOpts{});
    std::vector<int2> sizes(n);
    const int rc = round_trip(g, cu_stream, hf.data(), n, sizes.data(), n, [&](const PointFrame* d_in, int2* d_out, cudaStream_t st) {
        k->stmap_size<<<(unsigned)n, 128, 0, st>>>(d_in, (float)cp.width, (float)cp.height, d_out);
    });
    if (rc != GF_OK) return rc;
    size_t bad = n;
    for (size_t i = 0; i < n; ++i) {
        out_new_width[i] = sizes[i].x; out_new_height[i] = sizes[i].y;
        if (bad == n && !stmap_size_ok(sizes[i].x, sizes[i].y)) bad = i;
    }
    if (bad < n)
        return fail(nullptr, GF_ERR_SIZE_MISMATCH, "gf_cuda_stmap_sizes: undistorted frame size out of range: " + std::to_string(sizes[bad].x) + "x" +
                    std::to_string(sizes[bad].y) + " at entry " + std::to_string(bad) + " (frame " + std::to_string(frames[bad]) + ")");
    return GF_OK;
}

// zoom_dynamic::compute, static-window branch (zoom_dynamic.rs:56-76): sequential 1-D filters, stays on the host like in the reference
GF_API int gf_zoom_dynamic_compute(const double* fov_minimal, size_t n, double window_s, double fps, int method, double* out) {
    if (!fov_minimal || !out) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_zoom_dynamic_compute: null argument");
    if (n == 0) return GF_OK;
    std::vector<double> v(fov_minimal, fov_minimal + n);
    if (!zoom_static_window(v, window_s, fps, method)) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_zoom_dynamic_compute: zoom window longer than 1e8 frames");
    memcpy(out, v.data(), n * sizeof(double));
    return GF_OK;
}

GF_API int gf_zoom_fovs(const gf_zoom_params* zp, const double* timestamps_ms, const double* fov_values, size_t n,
                        double* out_fovs, double* out_minimal_fovs) {
    if (!zp) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_zoom_fovs: null argument");
    if (n == 0) return GF_OK;                                        // calculate_fovs returns empty vectors (zooming/mod.rs:36-38)
    if (!timestamps_ms || !fov_values || !out_fovs || !out_minimal_fovs || (zp->n_trim_ranges && !zp->trim_ranges))
        return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_zoom_fovs: null argument");
    std::vector<double> v(fov_values, fov_values + n);
    // Trim ranges (fov_iterative.rs:59-69) come before the mode branch, so the minimal FOVs of a trimmed clip carry the max-FOV fill.
    if (zp->n_trim_ranges > 0) {
        double max_fov = v[0];
        for (size_t i = 1; i < n; ++i) max_fov = fmax(max_fov, v[i]);                      // reduce(f64::max)
        const double l = (double)(n - 1);
        for (size_t i = 0; i < n; ++i) {
            bool within = false;
            for (size_t r = 0; r < zp->n_trim_ranges && !within; ++r)
                within = i >= as_usize(floor(l * zp->trim_ranges[2 * r])) && i <= as_usize(ceil(l * zp->trim_ranges[2 * r + 1]));
            if (!within) v[i] = max_fov;
        }
    }
    const std::vector<double> minimal = v;
    const double window = zp->adaptive_zoom_window, fps = zp->scaled_fps;
    const bool speed_keyed = track_keyed(zp->video_speed_track);
    if (window < -0.9) {                                             // static zoom (zooming/mod.rs:55-61)
        double m = v[0];
        for (size_t i = 1; i < n; ++i) m = fmin(m, v[i]);                                  // reduce(f64::min)
        v.assign(n, m);
    } else if (!(window > 0.0001)) {                                 // zoom disabled (:65-67)
        v.assign(n, 1.0);
    } else if (track_keyed(zp->zooming_speed) || (zp->video_speed_affects_zooming && (zp->video_speed != 1.0 || speed_keyed))) {   // zoom_dynamic.rs:22
        if (zp->adaptive_zoom_method == 1) {
            // The first envelope pass uses each frame's window (:26-30, :171-173); the second always 0.2 s (:51).
            std::vector<double> alphas(n);
            for (size_t i = 0; i < n; ++i) {
                double w = window, speed = zp->video_speed;
                (void)gf_keyframe_value_at(&zp->zooming_speed, timestamps_ms[i], zp->keyframe_timestamp_scale, &w);
                if (zp->video_speed_affects_zooming) {
                    (void)gf_keyframe_value_at(&zp->video_speed_track, timestamps_ms[i], zp->keyframe_timestamp_scale, &speed);
                    w *= fabs(speed);
                }
                alphas[i] = 1.0 - exp(-(1.0 / fps) / w);
            }
            v = envelope_follower(v, alphas);
            v = envelope_follower(v, std::vector<double>(n, 1.0 - exp(-(1.0 / fps) / 0.2)));
        } else {
            // get_frames_per_window reads the global adaptive_zoom_window, not the frame's window (zoom_dynamic.rs:31): every frame has the
            // static window, so min_rolling_dynamic / convolve_dynamic (:129-163) are the static min_rolling / convolve.
            if (!zoom_static_window(v, window, fps, 0)) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_zoom_fovs: zoom window longer than 1e8 frames");
        }
    } else if (!zoom_static_window(v, window, fps, zp->adaptive_zoom_method)) {                    // static window (zoom_dynamic.rs:56-76)
        return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_zoom_fovs: zoom window longer than 1e8 frames");
    }
    memcpy(out_fovs, v.data(), n * sizeof(double));
    memcpy(out_minimal_fovs, minimal.data(), n * sizeof(double));
    return GF_OK;
}

GF_API int gf_cuda_calculate_fovs(gf_cuda_gyro* g, const gf_compute_params* cp, const gf_zoom_params* zp, int distortion_model, int digital_lens,
                                  const double* timestamps_ms, size_t n, double* out_fovs, double* out_minimal_fovs, void* cu_stream) {
    if (!g || !cp || !zp || !timestamps_ms || !out_fovs || !out_minimal_fovs) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_calculate_fovs: null argument");
    if (n == 0) return GF_OK;
    std::vector<double> fov_values(n);
    const int rc = gf_cuda_find_fovs(g, cp, distortion_model, digital_lens, timestamps_ms, n, zp->fov_algorithm_margin, fov_values.data(), cu_stream);
    if (rc != GF_OK) return rc;
    return gf_zoom_fovs(zp, timestamps_ms, fov_values.data(), n, out_fovs, out_minimal_fovs);
}

GF_API int gf_cuda_sync_costs(gf_cuda_gyro* g, const gf_compute_params* cp, int distortion_model, int digital_lens, double scaled_fps,
                              const gf_sync_pair* pairs, size_t n_pairs, const double* offsets_ms, const double* readout_ms,
                              size_t n_candidates, int clear_offsets, double* out_costs, void* cu_stream) {
    int rc = sync_check("gf_cuda_sync_costs", g, cp, distortion_model, digital_lens, scaled_fps, pairs, n_pairs);
    if (rc != GF_OK) return rc;
    if (n_candidates && !out_costs) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_sync_costs: null argument");
    g->sync_host_ms = g->sync_device_ms = 0.0; g->sync_chunks = 0;
    if (n_candidates == 0) return GF_OK;
    CK(nullptr, cudaSetDevice(g->device));
    SyncJob J{ g, cp, distortion_model, scaled_fps, clear_offsets != 0, pairs, n_pairs, pick_kernels(distortion_model, digital_lens), g->stream_of(cu_stream) };
    if ((rc = sync_setup(J)) != GF_OK) return rc;
    return sync_run(J, offsets_ms, readout_ms, n_candidates, out_costs);
}

GF_API int gf_cuda_find_sync_offsets(gf_cuda_gyro* g, const gf_compute_params* cp, int distortion_model, int digital_lens, double scaled_fps,
                                     double initial_offset_ms, double search_size_ms, int for_rs,
                                     const gf_sync_range* ranges, size_t n_ranges, gf_sync_result* out, size_t* n_out, void* cu_stream) {
    int rc = sync_check("gf_cuda_find_sync_offsets", g, cp, distortion_model, digital_lens, scaled_fps, nullptr, 0);
    if (rc != GF_OK) return rc;
    if (!n_out || (n_ranges && (!ranges || !out))) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_find_sync_offsets: null argument");
    for (size_t r = 0; r < n_ranges; ++r)
        if ((rc = sync_check("gf_cuda_find_sync_offsets", g, cp, distortion_model, digital_lens, scaled_fps, ranges[r].pairs, ranges[r].n_pairs)) != GF_OK) return rc;
    *n_out = 0;
    g->sync_host_ms = g->sync_device_ms = 0.0; g->sync_chunks = 0;
    // the first stage: every 1 ms (:92-99, :118-125)
    std::vector<double> coarse;
    if (for_rs) {
        const double max_rs = 1000.0 / scaled_fps;
        if (max_rs >= kMaxSyncCandidates / 2) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_find_sync_offsets: more than 1e7 readout times (scaled_fps too small)");
        const int64_t steps = (int64_t)max_rs;                                   // `as isize`
        for (int64_t i = -steps; i < steps; ++i) coarse.push_back((double)i);
    } else if (search_size_ms >= kMaxSyncCandidates) {
        return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_find_sync_offsets: search_size of 1e7 ms or more");
    } else {
        const size_t steps = search_size_ms > 0.0 ? (size_t)search_size_ms : 0;       // `as usize` (NaN: 0)
        for (size_t i = 0; i < steps; ++i) coarse.push_back(initial_offset_ms + (-(search_size_ms / 2.0) + (double)i));
    }
    if (n_ranges == 0 || coarse.empty()) return GF_OK;
    CK(nullptr, cudaSetDevice(g->device));
    for (size_t r = 0; r < n_ranges; ++r) {
        const gf_sync_range& R = ranges[r];
        SyncJob J{ g, cp, distortion_model, scaled_fps, for_rs ? 0 : 1, R.pairs, R.n_pairs, pick_kernels(distortion_model, digital_lens), g->stream_of(cu_stream) };
        if ((rc = sync_setup(J)) != GF_OK) return rc;
        // offsets for the offset search, readout times (at offset 0) for the rolling-shutter estimate
        auto costs = [&](const std::vector<double>& cand, std::vector<double>& cost) {
            cost.assign(cand.size(), 0.0);
            return sync_run(J, for_rs ? nullptr : cand.data(), for_rs ? cand.data() : nullptr, cand.size(), cost.data());
        };
        std::vector<double> cost, fine(200), cost2;
        if ((rc = costs(coarse, cost)) != GF_OK) return rc;
        const double lowest = coarse[sync_last_min(cost)];
        for (int i = 0; i < 200; ++i) fine[i] = lowest - 1.0 + ((double)i * 0.01);          // then refine to 0.01 ms (:100-108, :126-134)
        if ((rc = costs(fine, cost2)) != GF_OK) return rc;
        const size_t b = sync_last_min(cost2);
        if (for_rs) { out[(*n_out)++] = gf_sync_result{ 0.0, fine[b], cost2[b] }; continue; }
        const double middle = ((double)R.from_us + (double)(int64_t)((uint64_t)R.to_us - (uint64_t)R.from_us) / 2.0) / 1000.0;   // :139
        if (fabs(fine[b] - initial_offset_ms) < search_size_ms * 0.9) out[(*n_out)++] = gf_sync_result{ middle, fine[b], cost2[b] };
    }
    return GF_OK;
}

GF_API int gf_cuda_sync_last_timing(const gf_cuda_gyro* g, double* host_record_ms, double* device_ms, size_t* chunks) {
    if (!g) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_sync_last_timing: null argument");
    if (host_record_ms) *host_record_ms = g->sync_host_ms;
    if (device_ms) *device_ms = g->sync_device_ms;
    if (chunks) *chunks = g->sync_chunks;
    return GF_OK;
}

} // extern "C"
