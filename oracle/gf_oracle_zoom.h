/* gf_oracle_zoom.h — CPU oracle of zooming::calculate_fovs after find_fov.  TEST INFRASTRUCTURE ONLY.
 *
 * A second module of the oracle (libgf_oracle_zoom.so, built by oracle/zoom.mk and linked against libgf_oracle.so, whose
 * gf_oracle_find_fov and gf_oracle_zoom_dynamic it calls).  Same float semantics as gf_oracle.h.  The product
 * (libgyroflow_cuda.so) never links or calls it.
 */
#ifndef GF_ORACLE_ZOOM_H
#define GF_ORACLE_ZOOM_H

#include "gf_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* zooming::calculate_fovs after find_fov: trim ranges (fov_iterative.rs:59-69), the zoom mode (zooming/mod.rs:55-68) and
 * zoom_dynamic::compute with both its branches (zoom_dynamic.rs:15-80).  The keyframe tracks of `zp` are not read: window[i] and
 * speed[i] are ZoomingSpeed / VideoSpeed at frame i's timestamp (adaptive_zoom_window / video_speed where the track has no key),
 * zooming_keyed / speed_keyed are is_keyframed of the two tracks. */
void gf_oracle_zoom_fovs(const gf_zoom_params* zp, const double* fov_values, const double* window, const double* speed,
                         int zooming_keyed, int speed_keyed, size_t n, double* out_fovs, double* out_minimal_fovs);
/* calculate_fovs (zooming/mod.rs:35-70) over n frames, frame index = position: gf_oracle_find_fov of every frame with the
 * adjustments of :41-49 and margin zp->fov_algorithm_margin, then gf_oracle_zoom_fovs.  `cp` is the user's ComputeParams. */
void gf_oracle_calculate_fovs(const gf_compute_params* cp, const gf_zoom_params* zp, int distortion_model, int digital_lens,
                              const double* timestamps_ms, const double* window, const double* speed, int zooming_keyed, int speed_keyed,
                              size_t n, double* out_fovs, double* out_minimal_fovs);

#ifdef __cplusplus
}
#endif
#endif
