/* gf_oracle_sync.h — CPU oracle of the visual-features sync search.  TEST INFRASTRUCTURE ONLY.
 *
 * A module of the oracle (libgf_oracle_sync.so, built by oracle/sync.mk and linked against libgf_oracle.so, whose
 * gf_oracle_undistort_points_rs_ex it calls): a literal restatement of find_offsets and its calculate_distance closure
 * (src/core/synchronization/find_offset/visual_features.rs:9-145), with a real sort of every pair's distances and the f64 sum in
 * ascending order.  Same float semantics as gf_oracle.h.  The product (libgyroflow_cuda.so) never links or calls it.
 * `threads` <= 0 means all online cores; the candidates of a stage are shared out like rayon's into_par_iter, and the minimum is
 * folded in candidate order afterwards, so the result does not depend on the thread count.
 */
#ifndef GF_ORACLE_SYNC_H
#define GF_ORACLE_SYNC_H

#include "gf_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* calculate_distance(offsets_ms[c], readout_ms ? Some(readout_ms[c]) : None) for every candidate c (offsets_ms NULL: 0), with the
 * gyro's sync offset cleared (gyro_offset_ms = 0, :12-15) when clear_offsets is set. */
void gf_oracle_sync_costs(const gf_compute_params* cp, int distortion_model, int digital_lens, double scaled_fps,
                          const gf_sync_pair* pairs, size_t n_pairs, const double* offsets_ms, const double* readout_ms,
                          size_t n_candidates, int clear_offsets, int threads, double* out_costs);
/* find_offsets over `ranges` (their pairs already selected); writes at most n_ranges results, returns how many. */
size_t gf_oracle_find_sync_offsets(const gf_compute_params* cp, int distortion_model, int digital_lens, double scaled_fps,
                                   double initial_offset_ms, double search_size_ms, int for_rs,
                                   const gf_sync_range* ranges, size_t n_ranges, int threads, gf_sync_result* out);

#ifdef __cplusplus
}
#endif
#endif
