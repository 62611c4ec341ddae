// frame_transform.cu — the producer of the warp's per-frame inputs, on the host and on the device.
//
// Behavioural source: FrameTransform::at_timestamp (src/core/stabilization/frame_transform.rs:165-350), get_frame_readout_time
// (:22-36), get_new_k (:37-51), get_fov (:52-58), focal_length_fov_compensation (:70-80), the IBIS / OIS row fill (:227-287 with
// CatmullRom::interpolate, gyro_source/splines.rs:22-83), per_frame_time_offsets (:224), GyroSource::quat_at_timestamp with
// multi-point sync offsets (src/core/gyro_source/mod.rs:857-909); quaternion algebra as nalgebra 0.34.2's UnitQuaternion<f64>
// (slerp, product, to_rotation_matrix) in quat_track.cuh; the rotation and shift of one row in frame_geometry.cuh.  All f64, narrowed to
// f32 at the very end (:300).  The per-frame host setup (keyframes, fov, K_new, readout timing, camera_stab) is shared with the point
// path of zoom_kernel.cu through c_abi_internal.h.
// Not evaluated here (they stay in Rust, see INTEGRATION.md "what stays on the Rust side"): keyframe curves (the caller passes
// the per-timestamp values in gf_compute_params), lens-profile interpolation (get_lens_data_at_timestamp: the caller passes the
// resulting camera matrix / coefficients), and mesh extraction from metadata (the caller passes mesh_data to the warp).
// The same row function is compiled for the host (gf_frame_transform_at_timestamp) and for the device
// (frame_rows_kernel: one thread per scanline).
#include <cuda_runtime.h>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/gyroflow_cuda.h"
#include "c_abi_internal.h"
#include "frame_geometry.cuh"

#define GF_FT_HD __host__ __device__ __forceinline__

using namespace gf;

namespace {

// everything per-frame-uniform the row function needs
struct RowCtx {
    Track org;
    SyncOffsets offsets;
    double duration_ms;
    Quat q0;                      // smoothed(ts) * org(ts)^-1   (:243-244,255-256)
    double rot_c, rot_s;          // image_rotation = Rz(video_rotation) (:241)
    double new_k[9];              // :37-51
    double start_ts, row_readout_time;
    int rs_on, framebuffer_inverted, suppress_rotation, zero_shifts;
    CameraStab stab;
};

// one scanline: frame_transform.rs:249-308
GF_FT_HD void frame_row(const RowCtx& C, size_t y, float* out14) {
    const double quat_time = C.rs_on ? C.start_ts + C.row_readout_time * (double)y : C.start_ts;       // :250-254
    const Quat qy = quat_at_timestamp(C.org, C.duration_ms, C.offsets, quat_time);
    const Quat q = qmul(C.q0, qy);                                                                     // :255-257
    double m[9];
    frame_rotation(q, C.rot_c, C.rot_s, C.new_k, C.framebuffer_inverted, C.suppress_rotation, m);      // :258-266,289-291
    // pinv(m): m is invertible (K_new has a positive focal length, r is a rotation up to sign flips) -> inverse via cofactors
    const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
    const double det = m[0] * c00 + m[1] * c01 + m[2] * c02;
    double inv[9] = { 0, 0, 0, 0, 0, 0, 0, 0, 0 };
    if (fabs(det) > 1e-300) {
        const double id = 1.0 / det;
        inv[0] = c00 * id;                          inv[1] = (m[2] * m[7] - m[1] * m[8]) * id; inv[2] = (m[1] * m[5] - m[2] * m[4]) * id;
        inv[3] = c01 * id;                          inv[4] = (m[0] * m[8] - m[2] * m[6]) * id; inv[5] = (m[2] * m[3] - m[0] * m[5]) * id;
        inv[6] = c02 * id;                          inv[7] = (m[1] * m[6] - m[0] * m[7]) * id; inv[8] = (m[0] * m[4] - m[1] * m[3]) * id;
    }
    for (int t = 0; t < 9; ++t) out14[t] = (float)inv[t];                                              // :300-304
    double sh[5] = { 0.0, 0.0, 0.0, 0.0, 0.0 };                                                        // :286
    if (C.stab.present) stab_shift(C.stab, (double)y, C.framebuffer_inverted, sh);                     // :269-285
    if (C.zero_shifts) { sh[0] = sh[1] = sh[2] = sh[3] = sh[4] = 0.0; }                                // :289-293 (suppress_rotation without rolling shutter)
    for (int t = 0; t < 5; ++t) out14[9 + t] = (float)sh[t];
}

// One thread per scanline.  The table's trust verdict (see warp_kernel_x2) is produced with it: every block ORs its rows into an
// accumulator, the last block to finish publishes the word and re-arms the accumulator and the ticket for the next launch, so no
// memset is needed and the verdict is ordered with the table on the producer's stream.
__global__ void frame_rows_kernel(const __grid_constant__ RowCtx C, size_t rows, float* __restrict__ out, uint32_t* __restrict__ flags_out,
                                  unsigned* __restrict__ scratch /* [0] accumulator, [1] ticket */) {
    const size_t y = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    unsigned f = 0;
    if (y < rows) {
        float row[14];
        frame_row(C, y, row);
        f = table_row_verdict(row);
        float2* o = reinterpret_cast<float2*>(out + y * GF_MATRIX_STRIDE);
        #pragma unroll
        for (int t = 0; t < 7; ++t) o[t] = make_float2(row[2 * t], row[2 * t + 1]);
    }
    if (!flags_out) return;
    __shared__ unsigned block_or;
    if (threadIdx.x == 0) block_or = 0u;
    __syncthreads();
    f = __reduce_or_sync(0xffffffffu, f);
    if ((threadIdx.x & 31u) == 0u && f) atomicOr(&block_or, f);
    __syncthreads();
    if (threadIdx.x == 0) {
        if (block_or) atomicOr(&scratch[0], block_or);
        __threadfence();
        if (atomicAdd(&scratch[1], 1u) == gridDim.x - 1u) {        // last block: every other block's OR is visible
            __threadfence();
            *flags_out = atomicExch(&scratch[0], 0u);
            scratch[1] = 0u;
        }
    }
}

// KeyframeManager::value_at_video_timestamp for one track — keyframes.rs:169-205 (without the custom_provider closure).
// Easing::get (keyframes.rs:279-291, sic: "b_in -> EaseOut", "a_out -> EaseIn") and Easing::interpolate (:292-302) with
// simple_easing 1.0.2's sine_in / sine_out / sine_in_out — easings.net: 1 - cos(x PI / 2), sin(x PI / 2), -(cos(PI x) - 1) / 2 — in f32
// through libm's cosf / sinf, like Rust's f32::cos / f32::sin on Linux.
bool keyframe_value(const gf_keyframe_track& t, double timestamp_ms, double scale, double* out) {
    if (!t.ts_us || !t.value || t.n == 0) return false;
    if (t.n == 1) { *out = t.value[0]; return true; }
    const double sc = scale != 0.0 ? scale : 1.0;
    const double r = round(timestamp_ms * 1000.0 * sc);                                        // f64::round, then `as i64` (saturating, NaN -> 0)
    const int64_t timestamp_us = r != r ? 0 : (r >= 9223372036854775807.0 ? INT64_MAX : (r <= -9223372036854775808.0 ? INT64_MIN : (int64_t)r));
    const int64_t first = t.ts_us[0], last = t.ts_us[t.n - 1];
    int64_t lookup = timestamp_us < last ? timestamp_us : last; if (lookup < first) lookup = first;     // .min(last_ts).max(first_ts)
    size_t lo = 0, hi = t.n;                                                                   // range(..=lookup).next_back(): last key <= lookup
    while (lo < hi) { const size_t mid = (lo + hi) / 2; if (t.ts_us[mid] <= lookup) lo = mid + 1; else hi = mid; }
    if (lo == 0) return false;
    const size_t i1 = lo - 1;
    if (t.ts_us[i1] == lookup) { *out = t.value[i1]; return true; }
    if (i1 + 1 >= t.n) return false;                                                           // range(lookup..).next()
    const size_t i2 = i1 + 1;
    const double time_delta = (double)(t.ts_us[i2] - t.ts_us[i1]);
    double x = (double)(timestamp_us - t.ts_us[i1]) / time_delta;
    const int ea = t.easing ? t.easing[i1] : 0, eb = t.easing ? t.easing[i2] : 0;
    const bool a_out = ea == 2 || ea == 3, b_in = eb == 1 || eb == 3;
    const int e = (a_out && b_in) ? 3 : (b_in ? 2 : (a_out ? 1 : 0));
    const float xf = (float)x, PI_F = 3.14159265358979323846f;
    if (e == 1)      x = (double)(1.0f - cosf(xf * PI_F / 2.0f));
    else if (e == 2) x = (double)sinf(xf * PI_F / 2.0f);
    else if (e == 3) x = (double)(-(cosf(PI_F * xf) - 1.0f) / 2.0f);
    *out = t.value[i1] * (1.0 - x) + t.value[i2] * x;
    return true;
}
// get_frame_readout_time — frame_transform.rs:22-36 (`scale` = capture_area_size.1 / sensor_size_px.1 of the closest lens_params
// entry, resolved by the caller into cp->readout_time_scale; 0 = no entry = 1.0)
double get_frame_readout_time(const gf_compute_params* cp, bool can_invert) {
    double t = fabs(cp->frame_readout_time);
    const double scale = cp->readout_time_scale != 0.0 ? cp->readout_time_scale : 1.0;
    if (can_invert && cp->framebuffer_inverted && !cp->readout_horizontal) t *= -1.0;
    if (cp->readout_inverted) t *= -1.0;
    return t * scale;
}

SyncOffsets host_offsets_of(const gf_compute_params* cp) {
    return SyncOffsets{ cp->sync_offset_ts_us, cp->sync_offset_ms, (cp->sync_offset_ts_us && cp->sync_offset_ms) ? cp->n_sync_offsets : 0, cp->gyro_offset_ms };
}

} // namespace

double gf::keyframed(const gf_compute_params* cp, int typ, double timestamp_ms, double dflt) {
    double v;
    return keyframe_value(cp->keyframes[typ], timestamp_ms, cp->keyframe_timestamp_scale, &v) ? v : dflt;
}

double gf::fov_unscaled(const gf_compute_params* cp, size_t frame, bool use_fovs, double timestamp_ms, bool for_ui) {
    double fov_scale = keyframed(cp, GF_KF_FOV, timestamp_ms, cp->fov_scale);
    fov_scale += (cp->fov_overview && use_fovs && !for_ui) ? 1.0 : 0.0;
    double fov = 1.0;
    if (use_fovs) {
        double f = 1.0;
        if (cp->fovs && frame < cp->n_fovs) f = cp->fovs[frame];
        else if (cp->fovs && cp->n_fovs > 1) f = cp->fovs[cp->n_fovs - 1];
        fov = f * fov_scale;
    }
    return fmax(fov, 0.001);
}

void gf::get_new_k(const gf_compute_params* cp, const double* camera_matrix, double fov, double (&new_k)[9]) {
    const double hr = cp->input_horizontal_stretch > 0.01 ? cp->input_horizontal_stretch : 1.0;     // :38 reads params.lens, the base profile
    const double img_dim_ratio = 1.0 / hr;
    memcpy(new_k, camera_matrix, sizeof(new_k));
    new_k[0] = new_k[0] * img_dim_ratio / fov; new_k[4] = new_k[4] * img_dim_ratio / fov;                   // :46-47
    new_k[2] = (double)cp->output_width / 2.0; new_k[5] = (double)cp->output_height / 2.0;                  // :48-49
}

gf::FrameTiming gf::frame_timing(const gf_compute_params* cp, size_t frame, double timestamp_ms, bool can_invert) {
    FrameTiming t;
    t.frame_readout_time = get_frame_readout_time(cp, can_invert);
    t.row_readout_time = t.frame_readout_time / (double)(cp->readout_horizontal ? cp->width : cp->height);
    if (cp->per_frame_time_offsets && frame < cp->n_per_frame_time_offsets) timestamp_ms += cp->per_frame_time_offsets[frame];
    t.start_ts = timestamp_ms - t.frame_readout_time / 2.0;
    const Track org{ cp->org.ts_us, cp->org.quats, cp->org.n }, sm{ cp->smoothed.ts_us, cp->smoothed.quats, cp->smoothed.n };
    const SyncOffsets ho = host_offsets_of(cp);
    const Quat quat1 = qinv(quat_at_timestamp(org, cp->duration_ms, ho, timestamp_ms));
    t.q0 = qmul(quat_at_timestamp(sm, cp->duration_ms, ho, timestamp_ms), quat1);
    return t;
}

gf::CameraStab gf::camera_stab_at(const gf_compute_params* cp, size_t frame, bool framebuffer_inverted, const StabSplines* splines) {
    CameraStab s; memset(&s, 0, sizeof(s));
    if (!cp->camera_stab || frame >= cp->n_camera_stab || !splines) return s;
    const gf_camera_stab& is = cp->camera_stab[frame];
    s.present = 1;
    s.offset = is.offset; s.sensor_h = (double)is.sensor_size[1];
    s.crop_y = (double)is.crop_area[1]; s.crop_h = (double)is.crop_area[3];
    s.height = (double)cp->height;
    s.scale_x = (double)cp->width  / (double)is.crop_area[2] / (double)is.pixel_pitch[0];
    s.scale_y = (double)cp->height / (double)is.crop_area[3] / (double)is.pixel_pitch[1] * (framebuffer_inverted ? -1.0 : 1.0);
    s.ibis = splines->ibis; s.ois = splines->ois;
    return s;
}

namespace {

// focal_length_fov_compensation — frame_transform.rs:70-80.  None is encoded as NaN (or any non-positive value, which the
// reference maps to 1.0 as well).
double focal_length_fov_compensation(const gf_compute_params* cp, size_t frame) {
    if (!cp->focal_length_smoothing_enabled) return 1.0;
    if (frame >= cp->n_focal_lengths || !cp->focal_lengths || !cp->smoothed_focal_lengths) return 1.0;
    const double dq = cp->focal_lengths[frame], sm = cp->smoothed_focal_lengths[frame];
    if (dq > 0.0 && sm > 0.0) return dq / sm;       // NaN compares false
    return 1.0;
}

// the per-frame-uniform part of at_timestamp: fills RowCtx (with the host tracks and sync offsets) + KernelParams, returns the number
// of rows.  `stab_splines`: the frame's spline points as the row function will address them (host pointers for the host producer, the
// uploaded copies for the device producer), or null when there are none.
size_t prepare(const gf_compute_params* cp, double timestamp_ms, size_t frame, const StabSplines* stab_splines,
               RowCtx& C, gf_kernel_params* kp, double* out_fov, double* out_minimal_fov) {
    // ----------- Keyframes :167-174 (evaluated at the frame's own timestamp, before per_frame_time_offsets) -----------
    const double video_rotation = keyframed(cp, GF_KF_VIDEO_ROTATION, timestamp_ms, cp->video_rotation);
    const double background_margin = keyframed(cp, GF_KF_BACKGROUND_MARGIN, timestamp_ms, cp->background_margin);
    const double background_feather = keyframed(cp, GF_KF_BACKGROUND_FEATHER, timestamp_ms, cp->background_margin_feather);
    const double lens_correction_amount = keyframed(cp, GF_KF_LENS_CORRECTION_STRENGTH, timestamp_ms, cp->lens_correction_amount);
    const double zoom_center_x = keyframed(cp, GF_KF_ZOOMING_CENTER_X, timestamp_ms, cp->adaptive_zoom_center_offset[0]);
    const double zoom_center_y = keyframed(cp, GF_KF_ZOOMING_CENTER_Y, timestamp_ms, cp->adaptive_zoom_center_offset[1]);
    const double light_refraction_coefficient = keyframed(cp, GF_KF_LIGHT_REFRACTION_COEFF, timestamp_ms, cp->light_refraction_coefficient);
    const double fl_compensation = focal_length_fov_compensation(cp, frame);                                              // :190
    const double size_ratio = (double)cp->width / (double)(cp->output_width > 1 ? cp->output_width : 1);                  // get_fov :56
    double fov = fov_unscaled(cp, frame, true, timestamp_ms, false) * size_ratio * fl_compensation;                       // :191
    double ui_fov = fov_unscaled(cp, frame, true, timestamp_ms, true) * size_ratio;
    if (cp->has_optimal_fov) { if (cp->n_fovs == 0) fov *= cp->lens_optimal_fov; else ui_fov /= cp->lens_optimal_fov; }   // :193-199
    // ----------- Lens :183-188: this frame's get_lens_data_at_timestamp result when the caller supplies one per frame -----------
    const gf_lens_data* lens = (cp->lens_per_frame && frame < cp->n_lens_per_frame) ? &cp->lens_per_frame[frame] : nullptr;
    const double* K = lens ? lens->camera_matrix : cp->camera_matrix;
    const double* dist = lens ? lens->distortion_coeffs : cp->distortion_coeffs;
    const double r_limit = lens ? lens->radial_distortion_limit : cp->radial_distortion_limit;
    const double ihs = lens ? lens->input_horizontal_stretch : cp->input_horizontal_stretch;
    const double ivs = lens ? lens->input_vertical_stretch : cp->input_vertical_stretch;
    const double hr_frame = ihs > 0.01 ? ihs : 1.0;                                                                     // :146 (the lens of this timestamp)

    const FrameTiming t = frame_timing(cp, frame, timestamp_ms, true);                                                   // :221-225,243-244
    const size_t n = (size_t)(cp->readout_horizontal ? cp->width : cp->height);
    const size_t rows = fabs(t.frame_readout_time) > 0.0 ? n : 1;                                                         // :247

    const double a = video_rotation * (M_PI / 180.0);
    C.org = Track{ cp->org.ts_us, cp->org.quats, cp->org.n }; C.duration_ms = cp->duration_ms; C.offsets = host_offsets_of(cp);
    C.q0 = t.q0;
    C.rot_c = cos(a); C.rot_s = sin(a);
    get_new_k(cp, K, fov, C.new_k);
    C.start_ts = t.start_ts; C.row_readout_time = t.row_readout_time;
    C.rs_on = fabs(t.frame_readout_time) > 0.0 ? 1 : 0;
    C.framebuffer_inverted = cp->framebuffer_inverted; C.suppress_rotation = cp->suppress_rotation;
    C.zero_shifts = (cp->suppress_rotation && cp->frame_readout_time == 0.0) ? 1 : 0;                                     // :289-293
    C.stab = camera_stab_at(cp, frame, cp->framebuffer_inverted, stab_splines);                                           // :227-236

    if (kp) {                                                                                                             // :322-340
        memset(kp, 0, sizeof(*kp));
        kp->matrix_count = (int32_t)rows;
        kp->f[0] = (float)K[0]; kp->f[1] = (float)K[4];
        kp->c[0] = (float)K[2]; kp->c[1] = (float)K[5];
        for (int i = 0; i < 12; ++i) kp->k[i] = (float)dist[i];
        kp->fov = (float)fov;
        kp->r_limit = (float)r_limit;
        kp->lens_correction_amount = (float)lens_correction_amount;
        kp->input_vertical_stretch = (float)(ivs > 0.01 ? ivs : 1.0);
        kp->input_horizontal_stretch = (float)hr_frame;
        kp->background_mode = cp->background_mode;
        kp->background_margin = (float)background_margin;
        kp->background_margin_feather = (float)background_feather;
        double zy = zoom_center_y;
        if (cp->framebuffer_inverted) zy *= -1.0;                                                                         // :318-320
        kp->translation2d[0] = (float)(zoom_center_x * (double)cp->width / fov);
        kp->translation2d[1] = (float)(zy * (double)cp->height / fov);
        for (int i = 0; i < cp->n_digital_lens_params && i < 16; ++i) kp->digital_lens_params[i] = (float)cp->digital_lens_params[i];
        kp->light_refraction_coefficient = (float)light_refraction_coefficient;
    }
    if (out_fov) *out_fov = ui_fov;                                                                                       // :345
    if (out_minimal_fov) *out_minimal_fov = frame < cp->n_minimal_fovs ? cp->minimal_fovs[frame] : 1.0;                   // :346
    return rows;
}

// One spline of a camera_stab entry.  A null position or value pointer means no points, whatever the count says: the host producer
// and the device upload read an entry the same way.
Spline3 stab_spline(const double* pos, const double* xyz, size_t n) {
    return Spline3{ pos, xyz, (pos && xyz) ? n : 0 };
}

// a device copy of n host values, into an empty buffer
template <class T> cudaError_t upload(GrowBuf<T>& d, const T* h, size_t n) {
    const cudaError_t e = d.reserve(n, nullptr);
    return e == cudaSuccess ? cudaMemcpy(d.ptr, h, n * sizeof(T), cudaMemcpyHostToDevice) : e;
}

} // namespace

#include "gyro_dev.h"

extern "C" {

GF_API int gf_keyframe_value_at(const gf_keyframe_track* track, double timestamp_ms, double timestamp_scale, double* out) {
    double v;
    if (!track || !keyframe_value(*track, timestamp_ms, timestamp_scale, &v)) return 0;
    if (out) *out = v;
    return 1;
}

GF_API int gf_frame_transform_at_timestamp(const gf_compute_params* cp, double timestamp_ms, size_t frame,
                                           gf_kernel_params* out_params, float* out_matrices, size_t max_rows,
                                           size_t* out_rows, double* out_fov, double* out_minimal_fov) {
    if (!cp || !out_matrices) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_frame_transform_at_timestamp: null argument");
    RowCtx C;
    StabSplines sp; memset(&sp, 0, sizeof(sp));
    if (cp->camera_stab && frame < cp->n_camera_stab) {
        const gf_camera_stab& is = cp->camera_stab[frame];
        sp.ibis = stab_spline(is.ibis_pos, is.ibis_xyz, is.n_ibis); sp.ois = stab_spline(is.ois_pos, is.ois_xyz, is.n_ois);
    }
    const size_t rows = prepare(cp, timestamp_ms, frame, &sp, C, out_params, out_fov, out_minimal_fov);
    if (out_rows) *out_rows = rows;
    if (rows > max_rows) return fail(nullptr, GF_ERR_BUFFER_TOO_SMALL, "gf_frame_transform_at_timestamp: max_rows below the frame's matrix rows");
    for (size_t y = 0; y < rows; ++y) frame_row(C, y, out_matrices + y * GF_MATRIX_STRIDE);       // rayon par_iter in the reference (:249)
    return GF_OK;
}

// Host-side form of the table verdict (what gf_cuda_frame_transform_dev leaves in table_flags_dev): 0 = tame and IBIS-free.
GF_API uint32_t gf_table_flags_host(const float* matrices, size_t rows) {
    uint32_t f = 0;
    if (matrices) for (size_t r = 0; r < rows; ++r) f |= table_row_verdict(matrices + r * GF_MATRIX_STRIDE);
    return f;
}

GF_API int gf_cuda_gyro_upload(gf_cuda_gyro** out, int device, const gf_compute_params* cp) {
    if (!out || !cp || !cp->org.ts_us || !cp->org.quats) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_gyro_upload: null argument");
    *out = nullptr;
    CK(nullptr, cudaSetDevice(device));
    std::unique_ptr<gf_cuda_gyro, Deleter<gf_cuda_gyro_free>> g(new gf_cuda_gyro());
    g->device = device; g->n_org = cp->org.n;
    CK(nullptr, upload(g->d_org_ts, cp->org.ts_us, cp->org.n));
    CK(nullptr, upload(g->d_org_q, cp->org.quats, cp->org.n * 4));
    CK(nullptr, create_stream(g->stream));
    CK(nullptr, g->d_scratch.reserve(2 * gf_cuda_gyro::kScratchPairs, nullptr));
    CK(nullptr, cudaMemset(g->d_scratch.ptr, 0, 2 * gf_cuda_gyro::kScratchPairs * sizeof(unsigned)));
    // multi-point sync offsets (offsets_adjusted) ride along with the tracks
    const SyncOffsets ho = host_offsets_of(cp);
    if (ho.n > 0) {
        g->n_offsets = ho.n;
        CK(nullptr, upload(g->d_off_ts, ho.ts, ho.n));
        CK(nullptr, upload(g->d_off_ms, ho.ms, ho.n));
    }
    // per-frame IBIS / OIS spline points (camera_stab_data): one flat device array + per-frame offsets kept on the host
    if (cp->camera_stab && cp->n_camera_stab > 0) {
        std::vector<double> flat;
        g->stab_index.resize(cp->n_camera_stab);
        for (size_t f = 0; f < cp->n_camera_stab; ++f) {
            const gf_camera_stab& is = cp->camera_stab[f];
            gf_cuda_gyro::StabIndex& ix = g->stab_index[f];
            ix.n_ibis = stab_spline(is.ibis_pos, is.ibis_xyz, is.n_ibis).n; ix.n_ois = stab_spline(is.ois_pos, is.ois_xyz, is.n_ois).n;
            ix.ibis_pos = flat.size(); flat.insert(flat.end(), is.ibis_pos, is.ibis_pos + ix.n_ibis);
            ix.ibis_val = flat.size(); flat.insert(flat.end(), is.ibis_xyz, is.ibis_xyz + 3 * ix.n_ibis);
            ix.ois_pos = flat.size();  flat.insert(flat.end(), is.ois_pos, is.ois_pos + ix.n_ois);
            ix.ois_val = flat.size();  flat.insert(flat.end(), is.ois_xyz, is.ois_xyz + 3 * ix.n_ois);
        }
        if (!flat.empty()) CK(nullptr, upload(g->d_stab, flat.data(), flat.size()));
    }
    // per-frame distorting meshes of the point path (mesh_correction[frame].0)
    if (cp->distorting_mesh && cp->n_distorting_mesh > 0) {
        std::vector<double> flat;
        g->mesh_index.resize(cp->n_distorting_mesh);
        for (size_t f = 0; f < cp->n_distorting_mesh; ++f) {
            const gf_mesh_f64& m = cp->distorting_mesh[f];
            gf_cuda_gyro::MeshIndex& ix = g->mesh_index[f];
            ix.off = flat.size(); ix.len = m.data ? m.len : 0;
            if (m.data) flat.insert(flat.end(), m.data, m.data + m.len);
            if (ix.len >= 9) memcpy(ix.header, m.data, sizeof(ix.header));
        }
        if (!flat.empty()) CK(nullptr, upload(g->d_mesh, flat.data(), flat.size()));
    }
    *out = g.release();
    return GF_OK;
}

GF_API void gf_cuda_gyro_free(gf_cuda_gyro* g) {
    if (!g) return;
    cudaSetDevice(g->device);
    if (g->stream) cudaStreamSynchronize(g->stream.get());
    if (g->stmap_done) cudaEventSynchronize(g->stmap_done.get());     // the last ST-map job, which may run on a caller's stream
    delete g;
    (void)cudaGetLastError();       // a failed teardown call must not fail the thread's next call
}

// `table_flags_dev` (nullable): receives the table's trust verdict on the same stream (see gf_cuda_undistort_image_dev_flagged).
// Stream ordering: with cu_stream == NULL the call runs on the gyro object's own stream and WAITS for it before returning (a
// consumer on any other stream may then read the table); with a stream it only enqueues — pass the same stream to the warp
// call, or order the two yourself.
GF_API int gf_cuda_frame_transform_dev_flagged(gf_cuda_gyro* g, const gf_compute_params* cp, double timestamp_ms, size_t frame,
                                               gf_kernel_params* out_params, float* matrices_dev, size_t max_rows, uint32_t* table_flags_dev,
                                               size_t* out_rows, double* out_fov, double* out_minimal_fov, void* cu_stream) {
    if (!g || !cp || !matrices_dev) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_frame_transform_dev_flagged: null argument");
    CK(nullptr, cudaSetDevice(g->device));
    RowCtx C;
    // the two per-frame lookups (org(ts), smoothed(ts)) stay on the host: O(log n) each; the per-row ones run on the device
    StabSplines sp;
    const bool has_stab = g->frame_splines(frame, sp);
    const size_t rows = prepare(cp, timestamp_ms, frame, has_stab ? &sp : nullptr, C, out_params, out_fov, out_minimal_fov);
    if (out_rows) *out_rows = rows;
    if (rows > max_rows) return fail(nullptr, GF_ERR_BUFFER_TOO_SMALL, "gf_cuda_frame_transform_dev_flagged: max_rows below the frame's matrix rows");
    C.org = g->org_track();
    C.offsets = g->sync_offsets(cp->gyro_offset_ms);
    const cudaStream_t st = g->stream_of(cu_stream);
    unsigned* scratch = g->d_scratch.ptr + 2u * (g->next_scratch++ % gf_cuda_gyro::kScratchPairs);     // self-cleaning: the last block re-arms it
    frame_rows_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, st>>>(C, rows, matrices_dev, table_flags_dev, scratch);
    CK(nullptr, cudaGetLastError());
    if (!cu_stream) CK(nullptr, cudaStreamSynchronize(st));
    return GF_OK;
}

GF_API int gf_cuda_frame_transform_dev(gf_cuda_gyro* g, const gf_compute_params* cp, double timestamp_ms, size_t frame,
                                       gf_kernel_params* out_params, float* matrices_dev, size_t max_rows,
                                       size_t* out_rows, double* out_fov, double* out_minimal_fov, void* cu_stream) {
    return gf_cuda_frame_transform_dev_flagged(g, cp, timestamp_ms, frame, out_params, matrices_dev, max_rows, nullptr, out_rows, out_fov, out_minimal_fov, cu_stream);
}

} // extern "C"
