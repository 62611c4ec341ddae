// frame_geometry.cuh — the per-frame gyro geometry both FrameTransform producers build on, host and device: the rotation of one
// row or point, the IBIS / OIS shift of one sensor row, and the frame-edge points of the FOV search.  frame_transform.cu
// (FrameTransform::at_timestamp, frame_transform.rs:165-350) and zoom_kernel.cu (at_timestamp_for_points, :352-438) both call
// these, so a row and a point at the same time get the same arithmetic.
#pragma once
#include "quat_track.cuh"

namespace gf {

// camera_stab_data[frame] resolved for one frame (frame_transform.rs:227-236, :412-418); spline points where the caller reads them
struct CameraStab {
    int present;
    double offset, sensor_h, crop_y, crop_h, scale_x, scale_y, height;
    Spline3 ibis, ois;
};
struct StabSplines { Spline3 ibis, ois; };

GF_QT_HD void mat3_mul(const double* a, const double* b, double* o) {
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) o[r * 3 + c] = a[r * 3 + 0] * b[0 * 3 + c] + a[r * 3 + 1] * b[1 * 3 + c] + a[r * 3 + 2] * b[2 * 3 + c];
}

// K_new * R for the rotation q: R = Rz(video rotation) * q.to_rotation_matrix() with the sign flips of the framebuffer orientation,
// or the identity under suppress_rotation — frame_transform.rs:258-266,289-291 (at_timestamp), :395-408 (at_timestamp_for_points,
// which always takes the framebuffer_inverted = false flips).
GF_QT_HD void frame_rotation(const Quat& q, double rot_c, double rot_s, const double* new_k, bool framebuffer_inverted, bool suppress_rotation,
                             double (&m)[9]) {
    // UnitQuaternion::to_rotation_matrix
    const double ww = q.w * q.w, ii = q.i * q.i, jj = q.j * q.j, kk = q.k * q.k;
    const double ij = q.i * q.j * 2.0, wk = q.w * q.k * 2.0, wj = q.w * q.j * 2.0, ik = q.i * q.k * 2.0, jk = q.j * q.k * 2.0, wi = q.w * q.i * 2.0;
    const double rq[9] = { ww + ii - jj - kk, ij - wk, wj + ik,
                           wk + ij, ww - ii + jj - kk, jk - wi,
                           ik - wj, wi + jk, ww - ii - jj + kk };
    const double rz[9] = { rot_c, -rot_s, 0.0, rot_s, rot_c, 0.0, 0.0, 0.0, 1.0 };
    double r[9];
    mat3_mul(rz, rq, r);
    if (framebuffer_inverted) { r[2] *= -1.0; r[5] *= -1.0; r[6] *= -1.0; r[7] *= -1.0; }
    else                      { r[1] *= -1.0; r[2] *= -1.0; r[3] *= -1.0; r[6] *= -1.0; }
    if (suppress_rotation) { for (int t = 0; t < 9; ++t) r[t] = (t % 4 == 0) ? 1.0 : 0.0; }
    mat3_mul(new_k, r, m);
}

// The IBIS / OIS shift of frame row `row` as (sx, sy, ra in radians, ox, oy) — frame_transform.rs:269-285 (at_timestamp), :419-429
// (at_timestamp_for_points, which never flips: framebuffer_inverted = false).  S must be present.
GF_QT_HD void stab_shift(const CameraStab& S, double row, bool framebuffer_inverted, double (&sh)[5]) {
    double y_sensor = (row - 0.0) * ((S.crop_y + S.crop_h) - S.crop_y) / (S.height - 0.0) + S.crop_y;   // map_coord, util.rs:144-147
    if (framebuffer_inverted) y_sensor = S.sensor_h - y_sensor;
    double v[3] = { 0.0, 0.0, 0.0 };
    if (!catmull_rom3(S.ibis, y_sensor + S.offset, v)) { v[0] = v[1] = v[2] = 0.0; }                   // unwrap_or_default
    sh[0] = v[0] * S.scale_x; sh[1] = v[1] * S.scale_y;
    const double ra = v[2] / 1000.0 * (framebuffer_inverted ? -1.0 : 1.0);
    sh[2] = ra * (3.14159265358979323846 / 180.0);                                                     // f64::to_radians
    double o[3] = { 0.0, 0.0, 0.0 };
    if (!catmull_rom3(S.ois, y_sensor + S.offset, o)) { o[0] = o[1] = o[2] = 0.0; }
    sh[3] = o[0] * S.scale_x; sh[4] = o[1] * S.scale_y;
}

// points_around_rect(w, h, 31, 31) with a margin, point k of RECT_POINTS — fov_iterative.rs:154-175
constexpr int RECT_POINTS = 120;
GF_QT_HD void rect_point(float w, float h, float margin, int k, float& x, float& y) {
    w -= margin * 2.0f; h -= margin * 2.0f;
    const int wcnt = 30, hcnt = 30;
    const float wstep = w / (float)wcnt, hstep = h / (float)hcnt;
    if (k < wcnt)                    { x = (float)k * wstep;                          y = 0.0f; }
    else if (k < wcnt + hcnt)        { x = w;                                         y = (float)(k - wcnt) * hstep; }
    else if (k < 2 * wcnt + hcnt)    { x = (float)(wcnt - (k - wcnt - hcnt)) * wstep; y = h; }
    else                             { x = 0.0f;                                      y = (float)(hcnt - (k - 2 * wcnt - hcnt)) * hstep; }
    x += margin; y += margin;
}

} // namespace gf
