// frame_params.cu — Stabilization::get_frame_transform_at<T> (src/core/stabilization/mod.rs:253-326) with get_kernel_flags
// (:226-251) and get_rect (:209-224): the per-buffer half of KernelParams, host only.
// FrameTransform::at_timestamp (frame_transform.cu) fills the per-timestamp half; this function completes the struct the way the
// reference does right before every process_pixels call, so that a Rust caller — or the render queue in this library — hands the
// warp exactly the bytes the reference's backends receive.
#include <cstring>
#include <cmath>
#include <cfloat>
#include "../../include/gyroflow_cuda.h"
#include "c_abi_internal.h"

namespace {

// T::COUNT, T::SCALAR_BYTES, T::default_max_value() — pixel_formats.rs:64-302
bool pixel_info(int pixel_type, int* count, int* scalar_bytes, float* max_value, bool* has_max) {
    *has_max = true;
    switch (pixel_type) {
    case GF_PIX_LUMA8:   *count = 1; *scalar_bytes = 1; *max_value = 255.0f;   return true;
    case GF_PIX_UV8:     *count = 2; *scalar_bytes = 1; *max_value = 255.0f;   return true;
    case GF_PIX_RGB8:    *count = 3; *scalar_bytes = 1; *max_value = 255.0f;   return true;
    case GF_PIX_RGBA8:
    case GF_PIX_BGRA8:   *count = 4; *scalar_bytes = 1; *max_value = 255.0f;   return true;
    case GF_PIX_LUMA16:  *count = 1; *scalar_bytes = 2; *max_value = 65535.0f; return true;
    case GF_PIX_UV16:    *count = 2; *scalar_bytes = 2; *max_value = 65535.0f; return true;
    case GF_PIX_RGB16:   *count = 3; *scalar_bytes = 2; *max_value = 65535.0f; return true;
    case GF_PIX_RGBA16:
    case GF_PIX_AYUV16:  *count = 4; *scalar_bytes = 2; *max_value = 65535.0f; return true;
    case GF_PIX_R32F:    *count = 1; *scalar_bytes = 4; *has_max = false;      return true;     // default_max_value() == None
    case GF_PIX_RGBAF:   *count = 4; *scalar_bytes = 4; *has_max = false;      return true;
    case GF_PIX_RGBAF16: *count = 4; *scalar_bytes = 2; *has_max = false;      return true;
    default: return false;
    }
}

void get_rect(const gf_buffer_desc* d, int32_t (&r)[4]) {                      // :209-224
    if (d->has_rect) { r[0] = d->rect[0]; r[1] = d->rect[1]; r[2] = d->rect[2]; r[3] = d->rect[3]; }
    else             { r[0] = 0; r[1] = 0; r[2] = d->width; r[3] = d->height; }   // stretch to the buffer by default
}

} // namespace

extern "C" GF_API int gf_get_frame_transform_at(const gf_stab_config* st, const gf_compute_params* cp, const gf_buffer_desc* in, const gf_buffer_desc* out,
                                                const float* mesh, size_t mesh_len, double timestamp_ms, size_t frame, double minimal_fov, gf_kernel_params* kp) {
    if (!st || !cp || !in || !out || !kp) return gf::fail(nullptr, GF_ERR_BAD_PARAMS, "gf_get_frame_transform_at: null argument");
    int count = 0, sbytes = 0; float maxv = 0.0f; bool has_max = false;
    if (!pixel_info(st->pixel_type, &count, &sbytes, &maxv, &has_max)) return gf::fail(nullptr, GF_ERR_BAD_PARAMS, "gf_get_frame_transform_at: unknown pixel type");

    kp->pixel_value_limit = has_max ? maxv : FLT_MAX;                           // :258 T::default_max_value().unwrap_or(f32::MAX)
    kp->max_pixel_value   = has_max ? maxv : 1.0f;                              // :259
    kp->interpolation = st->interpolation;                                      // :265
    kp->width = st->width; kp->height = st->height;                             // :266-267
    kp->output_width = st->output_width; kp->output_height = st->output_height; // :268-269
    for (int i = 0; i < 4; ++i) kp->background[i] = st->background[i];          // :270
    kp->bytes_per_pixel = count * sbytes;                                       // :271
    kp->pix_element_count = count;                                              // :272
    kp->canvas_scale = st->canvas_scale;                                        // :273

    // get_kernel_flags :226-251
    int32_t flags = st->base_flags & (GF_FLAG_FIX_COLOR_RANGE | GF_FLAG_FILL_WITH_BACKGROUND | GF_FLAG_DRAWING_ENABLED);
    if (st->has_digital_lens) flags |= GF_FLAG_HAS_DIGITAL_LENS;
    if (cp->readout_horizontal) flags |= GF_FLAG_HORIZONTAL_RS;
    if (in->has_rect || st->width != in->width || st->height != in->height) flags |= GF_FLAG_HAS_SOURCE_RECT;
    if (out->has_rect || st->output_width != out->width || st->output_height != out->height) flags |= GF_FLAG_HAS_OUTPUT_RECT;
    if (cp->framebuffer_inverted) flags |= GF_FLAG_FRAMEBUFFER_INVERTED;
    if ((cp->light_refraction_coefficient != 1.0 && cp->light_refraction_coefficient > 0.0) || st->light_refraction_keyframed) flags |= GF_FLAG_ANY_UNDERWATER;
    if (mesh && mesh_len > 0) {                                                 // file_metadata.mesh_correction.get(frame)
        if (mesh[0] > 10.0f) flags |= GF_FLAG_HAS_MESH_DATA;
        // `mc.1[mc.1[0] as usize] > 0.0`: the reference indexes unchecked (a mesh without the focal-plane block would panic)
        const float m0 = mesh[0];
        const size_t o = m0 != m0 ? 0 : (m0 <= 0.0f ? 0 : (size_t)m0);
        if (m0 > 0.0f && o < mesh_len && mesh[o] > 0.0f) flags |= GF_FLAG_HAS_FPD_DATA;
    }
    if (st->has_ibis_data || (cp->camera_stab && cp->n_camera_stab > frame)) flags |= GF_FLAG_HAS_IBIS_DATA;
    kp->flags = flags;                                                          // :274

    kp->stride = in->stride;                                                    // :276-277
    kp->output_stride = out->stride;

    if (kp->interpolation > 8) {                                                // :279-295, f32 arithmetic
        float b = 0.0f, c = 0.0f;
        switch (kp->interpolation) {
        case GF_INTERP_ROBIDOUX_SHARP: b = 0.2620145f; c = 0.3689927f; break;
        case GF_INTERP_ROBIDOUX:       b = 0.3782157f; c = 0.3108921f; break;
        case GF_INTERP_MITCHELL:       b = 0.3333333f; c = 0.3333333f; break;
        case GF_INTERP_CATMULL_ROM:    b = 0.0000000f; c = 0.5000000f; break;
        default: break;
        }
        kp->ewa_coeffs_p[0] = (6.0f - 2.0f * b) / 6.0f;
        kp->ewa_coeffs_p[1] = 0.0f;
        kp->ewa_coeffs_p[2] = (-18.0f + 12.0f * b + 6.0f * c) / 6.0f;
        kp->ewa_coeffs_p[3] = (12.0f - 9.0f * b - 6.0f * c) / 6.0f;
        kp->ewa_coeffs_q[0] = (8.0f * b + 24.0f * c) / 6.0f;
        kp->ewa_coeffs_q[1] = (-12.0f * b - 48.0f * c) / 6.0f;
        kp->ewa_coeffs_q[2] = (6.0f * b + 30.0f * c) / 6.0f;
        kp->ewa_coeffs_q[3] = (-1.0f * b - 6.0f * c) / 6.0f;
    }

    float sa_fov = 1.0f;                                                        // :297-308
    if (st->show_safe_area || cp->fov_overview) {
        double kf_fov = cp->fov_scale;                                          // keyframes.value_at_video_timestamp(Fov, ts).unwrap_or(fov_scale)
        (void)gf_keyframe_value_at(&cp->keyframes[GF_KF_FOV], timestamp_ms, cp->keyframe_timestamp_scale, &kf_fov);
        const float fov = (float)kf_fov;
        if (cp->fov_overview) sa_fov = (st->adaptive_zoom_window == 0.0 ? 1.0f : 1.0f / fov) + 1.0f;
        else                  sa_fov = fov / (st->adaptive_zoom_window == 0.0 ? (float)minimal_fov : 1.0f);
    }
    const float ow = (float)kp->output_width, oh = (float)kp->output_height;
    const float pos_x = (ow - (ow / sa_fov)) / 2.0f;                            // :309-314
    const float pos_y = (oh - (oh / sa_fov)) / 2.0f;
    kp->safe_area_rect[0] = pos_x; kp->safe_area_rect[1] = pos_y;
    kp->safe_area_rect[2] = ow - pos_x; kp->safe_area_rect[3] = oh - pos_y;

    if (in->has_rotation)  kp->input_rotation  = in->rotation;                  // :316-321
    if (out->has_rotation) kp->output_rotation = out->rotation;
    get_rect(in,  kp->source_rect);                                             // :322-323
    get_rect(out, kp->output_rect);
    return GF_OK;
}
