"""ST maps (SURVEY f4): gf_cuda_generate_stmap against generate_stmaps (src/core/stmap.rs:6-146) restated with the oracle's pieces."""
import copy
import ctypes as C

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi
from tests import oracle_lib
from tests.test_zoom import make_cp

F = np.float32


def oracle_stmap(cp, lens, digital, ts, frame, per_frame):
    """stmap.rs:24-116 with the oracle: returns (new_w, new_h, dist, undist); no maps (None) for an undistorted size the product
    refuses."""
    lib = oracle_lib.load()
    m, d = abi.LENS[lens], abi.LENS[digital] if digital else 0
    c = cp.c
    w, h = c.width, c.height
    saved = (c.frame_readout_time, c.suppress_rotation, c.fovs, c.n_fovs, c.fov_scale, c.output_width, c.output_height)
    try:
        if not per_frame: c.frame_readout_time = 0.0
        c.suppress_rotation = 1; c.n_fovs = 0
        c.fov_scale = 1.0; c.output_width, c.output_height = w, h
        # points_around_rect(w, h, 31, 31), margin 0 (fov_iterative.rs:154-175)
        wstep, hstep = F(w) / F(30), F(h) / F(30)
        rect = [(F(i) * wstep, F(0)) for i in range(30)] + [(F(w), F(i) * hstep) for i in range(30)] + \
               [(F(30 - i) * wstep, F(h)) for i in range(30)] + [(F(0), F(30 - i) * hstep) for i in range(30)]
        pts = np.array(rect, dtype=np.float32)
        und = np.zeros_like(pts)
        lib.gf_oracle_undistort_points_rs_ex(C.byref(c), m, d, pts.ctypes.data, len(pts), ts, frame, 1.0, 0, und.ctypes.data)
        min_x = min(F(0), und[:, 0].min()); min_y = min(F(0), und[:, 1].min())
        max_x = max(F(0), und[:, 0].max()); max_y = max(F(0), und[:, 1].max())
        new_w = int(np.ceil(F(max_x - min_x))); new_h = int(np.ceil(F(max_y - min_y)))
        # gf_cuda_generate_stmap refuses these sizes: beyond 32768, and wider than the 16384 the warp that renders the undistort map takes
        if not (4 <= new_w <= 16384 and 4 <= new_h <= 32768):
            return new_w, new_h, None, None
        c.fov_scale = float(max(F(new_w) / F(w), F(new_h) / F(h)))
        c.width = c.output_width = new_w; c.height = c.output_height = new_h
        kp, mats, _, _ = cp.at_timestamp(ts, frame)                        # the product's host producer (tests/test_frame_transform.py)
        kp.width = kp.output_width = new_w; kp.height = kp.output_height = new_h
        kp.flags = (abi.FLAG_HAS_DIGITAL_LENS if digital else 0) | (abi.FLAG_HORIZONTAL_RS if c.readout_horizontal else 0)
        undist = np.zeros((new_h, new_w, 3), np.float32)
        mats = np.ascontiguousarray(mats, dtype=np.float32)
        lib.gf_oracle_stmap_undistort(C.byref(kp), mats.ctypes.data, m, d, undist.ctypes.data)
        c.width = c.output_width = w; c.height = c.output_height = h
        dist = np.zeros((h, w, 3), np.float32)
        lib.gf_oracle_stmap_distort(C.byref(c), m, d, ts, frame, dist.ctypes.data)
        return new_w, new_h, dist, undist
    finally:
        c.frame_readout_time, c.suppress_rotation, c.fovs, c.n_fovs, c.fov_scale, c.output_width, c.output_height = saved
        c.width, c.height = w, h


def test_oracle_stmap_identity_lens_is_the_identity_map():
    """No distortion, no rotation: both maps are (x / w, 1 - y / h, 0) and the undistorted size equals the frame size."""
    cp = make_cp(w=96, h=54)
    cp.c.distortion_coeffs[:] = [0.0] * 12
    nw, nh, dist, und = oracle_stmap(cp, "opencv_fisheye", None, 500.0, 30, False)
    assert (nw, nh) == (96, 54)
    xs, ys = np.meshgrid(np.arange(96, dtype=np.float32), np.arange(54, dtype=np.float32))
    for mp in (dist, und):
        assert np.allclose(mp[..., 0], xs / 96, atol=2e-4) and np.allclose(mp[..., 1], 1 - ys / 54, atol=2e-4) and (mp[..., 2] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("lens,digital,per_frame,kw", [
    ("opencv_fisheye", None, True, {}),
    ("opencv_fisheye", None, False, {}),
    ("opencv_fisheye", "gopro_superview", True, {}),
    ("sony", None, True, {}),
    ("opencv_standard", "digital_stretch", True, dict(horizontal=True)),
    ("gopro", "gopro_warp", False, {}),
])
def test_generate_stmap_matches_oracle(lens, digital, per_frame, kw):
    cp = make_cp(w=240, h=136, lens=lens, digital=digital, **dict(kw))
    ts, frame = 1000.0 / 60.0 * 40, 40
    nw, nh, want_dist, want_und = oracle_stmap(cp, lens, digital, ts, frame, per_frame)
    dg = g.DeviceGyro(cp)
    dist, und = dg.generate_stmap(lens, digital, ts, frame, per_frame)
    dg.close()
    assert und.shape == (nh, nw, 3) and dist.shape == (136, 240, 3)
    assert np.array_equal(und, want_und), "undistort map differs: %d values" % int((und != want_und).sum())
    # generate_stmap suppresses the rotation (stmap.rs:28-34), so no f64 libm result reaches the redistort map: bit for bit, and two
    # NaNs count as equal whatever their payload (the host's default NaN is not the GPU's)
    same = (dist.view(np.uint32) == want_dist.view(np.uint32)) | (np.isnan(dist) & np.isnan(want_dist))
    assert same.all(), "redistort map differs: %d values" % int((~same).sum())


def test_oracle_stmap_matches_second_restatement():
    """generate_stmaps (stmap.rs:24-136) for opencv_fisheye with the SECOND transcriptions: the undistort map from
    tests/np_restatement.rotate_and_distort + the rolling-shutter row pick of :88-109, the redistort map from
    tests/np_zoom.undistort_points_with_rolling_shutter(use_fovs = true), both in the (x / w, 1 - y / h, 0) encoding of :131-135 —
    against the oracle's maps.  The undistort map is byte-identical given the same matrices, and so is the redistort map: its rotation
    is suppressed."""
    import warnings
    from tests import np_restatement as npr, np_zoom
    for per_frame in (True, False):
        cp = make_cp(w=64, h=36)
        ts, frame = 1000.0 / 60.0 * 40, 40
        nw, nh, want_dist, want_und = oracle_stmap(cp, "opencv_fisheye", None, ts, frame, per_frame)
        # ---- the state generate_stmaps leaves compute_params in for each map (:28-34, :73-76, :112-113) ----
        c = cp.c
        w, h = c.width, c.height
        saved = (c.frame_readout_time, c.suppress_rotation, c.n_fovs, c.fov_scale)
        if not per_frame: c.frame_readout_time = 0.0
        c.suppress_rotation = 1; c.n_fovs = 0
        c.fov_scale = float(max(F(nw) / F(w), F(nh) / F(h)))
        c.width = c.output_width = nw; c.height = c.output_height = nh
        kp, mats, _, _ = cp.at_timestamp(ts, frame)
        kp.width = kp.output_width = nw; kp.height = kp.output_height = nh
        kp.flags = 0
        m = [[F(v) for v in row] for row in np.asarray(mats, dtype=np.float32)]
        got_und = np.zeros((nh, nw, 3), np.float32)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for yi in range(nh):
                for xi in range(nw):
                    x, y = F(xi), F(yi)
                    sy = max(min(npr.as_i32(npr.round_half_away(y)), kp.height), 0)
                    if kp.matrix_count > 1:
                        pt = npr.rotate_and_distort(x, y, kp.matrix_count // 2, kp, m)
                        if pt is not None:
                            sy = max(min(npr.as_i32(npr.round_half_away(pt[1])), kp.height), 0)
                    uv = npr.rotate_and_distort(x, y, min(sy, kp.matrix_count - 1), kp, m) or (F(0.0), F(0.0))
                    got_und[yi, xi] = (uv[0] / F(nw), F(1.0) - (uv[1] / F(nh)), 0.0)
            assert np.array_equal(got_und, want_und)
            c.width = c.output_width = w; c.height = c.output_height = h
            got_dist = np.zeros((h, w, 3), np.float32)
            for yi in range(0, h, 5):                                      # every 5th row keeps the pure-Python loop short
                for xi in range(w):
                    (ux, uy), = np_zoom.undistort_points_with_rolling_shutter(cp, [(F(xi), F(yi))], ts, frame, 1.0, use_fovs=True)
                    got_dist[yi, xi] = (ux / F(w), F(1.0) - (uy / F(h)), 0.0)
            assert np.array_equal(got_dist[::5], want_dist[::5])
        c.frame_readout_time, c.suppress_rotation, c.n_fovs, c.fov_scale = saved
