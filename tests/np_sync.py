"""Second, independent restatement of the visual-features sync search — TEST INFRASTRUCTURE ONLY.

  calculate_distance / find_offsets   <- src/core/synchronization/find_offset/visual_features.rs:9-145
  frame_at_timestamp                  <- src/core/lib.rs:2069

Written from the Rust text on tests/np_zoom.py's point path; the C oracle (oracle/gf_oracle_sync.c) and the CUDA kernel
(sync_cost_kernel in gyroflow_b200/csrc/zoom_kernel.cu) are checked against it in tests/test_sync_offsets.py.  np_zoom's point path
reads no gyro sync offset, which is what the offset search sees (it clears them); the rolling-shutter estimate keeps them, so it is
restated here for a ComputeParams without one.
A pair is ((ts_us, pts1), (next_ts_us, pts2)) with (n, 2) float32 point lists; `stabs` / `meshes` are the clip's per-frame CameraStab
dicts and distorting meshes (as given to backend.ComputeParams), looked up by the frame of each timestamp.
"""
import math

import numpy as np

from tests import np_zoom

F32 = np.float32


def f64_round(x):
    """f64::round: half away from zero (Python's round() rounds half to even)."""
    t = math.trunc(x)
    if abs(x - t) >= 0.5:
        t += 1 if x > 0 else -1
    return t


def frame_at_timestamp(timestamp_ms, fps):
    """`frame_at_timestamp(ts, fps) as usize`: round, `as i32` (saturating), then a negative value wraps through usize."""
    v = timestamp_ms * (fps / 1000.0)
    i = 0 if v != v else max(-2 ** 31, min(2 ** 31 - 1, f64_round(v)))
    return i % 2 ** 64


def undistort(cp, pts, timestamp_ms, fps, lens, digital, stabs, meshes):
    """undistort_points_with_rolling_shutter(pts, timestamp_ms, None, params, 1.0, false) — cpu_undistort.rs:636-641."""
    frame = frame_at_timestamp(timestamp_ms, fps)
    stab = stabs[frame] if stabs and frame < len(stabs) else None
    mesh = meshes[frame] if meshes and frame < len(meshes) else None
    mesh = None if mesh is None else [float(v) for v in mesh]
    return np_zoom.undistort_points_with_rolling_shutter(cp, [tuple(p) for p in pts], timestamp_ms, frame, 1.0, False, lens, digital, stab, mesh)


def calculate_distance(cp, pairs, offs, rs, fps, lens, digital, stabs=None, meshes=None, points=None):
    """visual_features.rs:46-84; rs None: the ComputeParams' own frame_readout_time.  points(pts, timestamp_ms): another point path to
    compose the cost from (it sees `cp` with the candidate's readout time); default np_zoom's."""
    points = points or (lambda pts, t: undistort(cp, pts, t, fps, lens, digital, stabs, meshes))
    c = cp.c
    saved = c.frame_readout_time
    if rs is not None:
        c.frame_readout_time = rs
    try:
        w, h = F32(c.width), F32(c.height)
        total = 0.0
        for (ts, pts1), (next_ts, pts2) in pairs:
            if len(pts1) == 0:
                continue
            t1, t2 = ts / 1000.0, next_ts / 1000.0
            u1 = points(np.asarray(pts1, np.float32), t1 - offs)
            u2 = points(np.asarray(pts2, np.float32), t2 - offs)
            distances = []
            for (x1, y1), (x2, y2) in zip(u1, u2):
                x1, y1, x2, y2 = F32(x1), F32(y1), F32(x2), F32(y2)
                if x1 > 0 and x1 < w and y1 > 0 and y1 < h and x2 > 0 and x2 < w and y2 > 0 and y2 < h:
                    dist = ((x2 - x1) * (x2 - x1)) + ((y2 - y1) * (y2 - y1))         # f32
                    distances.append(int(dist))                                        # `as u64` of a finite, non-negative f32
            distances.sort()
            for d in distances[:int(len(distances) * 0.9)]:
                total += float(d)
        return total
    finally:
        c.frame_readout_time = saved


def _no_offsets(cp):
    return cp.c.gyro_offset_ms == 0.0 and cp.c.n_sync_offsets == 0


def sync_costs(cp, pairs, offsets_ms, readout_ms, fps, lens, digital, stabs=None, meshes=None, points=None):
    assert points or readout_ms is None or _no_offsets(cp), "np_zoom's point path reads no sync offset"
    n = len(offsets_ms) if offsets_ms is not None else len(readout_ms)
    return np.array([calculate_distance(cp, pairs, offsets_ms[i] if offsets_ms is not None else 0.0,
                                        readout_ms[i] if readout_ms is not None else None, fps, lens, digital, stabs, meshes, points)
                     for i in range(n)])


def find_min(cands):
    """reduce_with(find_min): `if a.1 < b.1 { a } else { b }` over the candidates in order."""
    best = cands[0]
    for x in cands[1:]:
        best = best if best[1] < x[1] else x
    return best


def find_offsets(cp, ranges, initial_offset, search_size, for_rs, fps, lens, digital, stabs=None, meshes=None):
    """visual_features.rs:9-145 over [(from_us, to_us, pairs)]: [(timestamp_ms, value_ms, cost)]."""
    assert not for_rs or _no_offsets(cp), "np_zoom's point path reads no sync offset"
    final = []
    for from_ts, to_ts, pairs in ranges:
        dist = lambda v: calculate_distance(cp, pairs, 0.0 if for_rs else v, v if for_rs else None, fps, lens, digital, stabs, meshes)
        if for_rs:
            max_rs = 1000.0 / fps
            steps = int(max_rs)                                                        # `as isize`
            coarse = [float(i) for i in range(-steps, steps)]
        else:
            steps = int(search_size) if search_size > 0 else 0                         # `as usize`
            coarse = [initial_offset + (-(search_size / 2.0) + float(i)) for i in range(steps)]
        if not coarse:
            continue
        lowest = find_min([(v, dist(v)) for v in coarse])
        lowest = find_min([(v, dist(v)) for v in (lowest[0] - 1.0 + (i * 0.01) for i in range(200))])
        if for_rs:
            final.append((0.0, lowest[0], lowest[1]))
        else:
            middle = (float(from_ts) + float(to_ts - from_ts) / 2.0) / 1000.0
            if abs(lowest[0] - initial_offset) < search_size * 0.9:
                final.append((middle, lowest[0], lowest[1]))
    return final
