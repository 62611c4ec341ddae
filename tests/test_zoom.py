"""Adaptive-zoom companion (SURVEY §8 a17): FovIterative::find_fov + zoom_dynamic."""
import ctypes as C

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi, synth
from tests import cases, oracle_lib


def make_cp(w=1920, h=1080, ow=None, oh=None, lens="opencv_fisheye", digital=None, **kw):
    p = synth.base_kernel_params(w, h, ow, oh, lens=lens, digital_lens=digital)
    for k, v in kw.pop("params", {}).items():
        setattr(p, k, v)
    org, sm = cases.gyro()
    return g.ComputeParams(p, org, sm, **kw)


def test_oracle_fov_properties():
    ts = np.arange(30) * (1000.0 / 60.0)
    # identity lens, no rotation: the whole frame (minus the 2 px margin) is visible -> fov just below 1
    cp = make_cp(params=dict())
    cp.c.distortion_coeffs[:] = [0.0] * 12
    cp.c.suppress_rotation = 1
    f = oracle_lib.find_fovs(cp, "opencv_fisheye", None, ts)
    assert np.allclose(f, (1920 - 4) / 1920.0, atol=2e-3)
    # with the synthetic shake the fov varies frame to frame and stays in a sane range
    f2 = oracle_lib.find_fovs(make_cp(), "opencv_fisheye", None, ts)
    assert f2.std() > 1e-3 and 0.5 < f2.min() and f2.max() < 1.5


def test_zoom_dynamic_host_matches_oracle_bit_for_bit():
    rng = np.random.default_rng(3)
    fm = 0.9 + 0.1 * rng.random(400)
    for method in (0, 1):
        a = g.zoom_dynamic(fm, 4.0, 60.0, method)
        b = oracle_lib.zoom_dynamic(fm, 4.0, 60.0, method)
        assert np.array_equal(a, b)
        assert (a <= fm + 1e-12).all() if method == 1 else a.shape == fm.shape      # the envelope never exceeds the per-frame minimum
        from tests import np_zoom
        assert np.array_equal(a, np.asarray(np_zoom.zoom_dynamic(fm, 4.0, 60.0, method)))       # second transcription (zoom_dynamic.rs:56-76)
    for window_s, fps in ((0.5, 29.97), (2.0, 24.0)):                            # even / odd window lengths
        for method in (0, 1):
            assert np.array_equal(g.zoom_dynamic(fm[:97], window_s, fps, method), np.asarray(np_zoom.zoom_dynamic(fm[:97], window_s, fps, method)))


@pytest.mark.gpu
@pytest.mark.parametrize("lens,digital,kw", [
    ("opencv_fisheye", None, {}),
    ("opencv_fisheye", "gopro_superview", {}),
    ("sony", None, {}),
    ("gopro", "gopro_warp", {}),
    ("opencv_standard", "digital_stretch", {}),
    ("opencv_fisheye", None, dict(ow=1280, oh=720)),
    ("opencv_fisheye", None, dict(frame_readout_time_ms=0.0)),
    ("opencv_fisheye", None, dict(video_rotation=12.0, horizontal=True)),
    ("opencv_fisheye", "gopro_superview", dict(params=dict(lens_correction_amount=0.4))),
    ("poly5", None, dict(params=dict(lens_correction_amount=0.7))),
])
def test_device_find_fovs_matches_oracle(lens, digital, kw):
    cp = make_cp(lens=lens, digital=digital, **dict(kw))
    ts = np.arange(120) * (1000.0 / 60.0)
    want = oracle_lib.find_fovs(cp, lens, digital, ts)
    dg = g.DeviceGyro(cp)
    got = dg.find_fovs(lens, digital, ts)
    dg.close()
    assert np.allclose(got, want, rtol=1e-6, atol=0), float(np.abs(got / want - 1).max())
    assert (got == want).mean() > 0.9            # almost always identical; the rest is f64 device-vs-host libm in the rotation


@pytest.mark.gpu
def test_device_find_fovs_with_keyframes_matches_oracle_per_frame():
    """Keyframed clips (fov_iterative.rs:41-52): every frame uses ITS zoom centre and lens-correction strength, and the point path its video
    rotation (frame_transform.rs:354) and refraction coefficient (cpu_undistort.rs:661).  The device result for frame i equals the oracle's
    find_fov on a ComputeParams whose constants are the restated KeyframeManager's values at that frame's timestamp."""
    from tests import np_producer
    tracks = {"VideoRotation": [(0, -8.0, "EaseInOut"), (900_000, 14.0, "EaseOut"), (2_000_000, 3.0, "NoEasing")],
              "ZoomingCenterX": [(100_000, -0.04, "EaseIn"), (1_500_000, 0.05, "EaseInOut")],
              "ZoomingCenterY": [(0, 0.03, "NoEasing"), (1_900_000, -0.02, "EaseOut")],
              "LensCorrectionStrength": [(0, 1.0, "EaseInOut"), (1_000_000, 0.35, "EaseInOut"), (2_000_000, 0.8, "EaseIn")],
              "LightRefractionCoeff": [(0, 1.0, "NoEasing"), (2_000_000, 1.33, "NoEasing")]}
    lens, digital = "opencv_fisheye", None
    cp = make_cp(lens=lens, digital=digital, keyframes=tracks)
    ts = np.arange(0, 120, 3) * (1000.0 / 60.0)
    dg = g.DeviceGyro(cp)
    got = dg.find_fovs(lens, digital, ts)
    # single-timestamp point path: rotation / refraction resolved at the timestamp
    pts = np.array([[100.0, 80.0], [960.0, 540.0], [1800.0, 1000.0]], np.float32)
    got_pts = dg.undistort_points(lens, digital, pts, float(ts[7]))
    dg.close()
    want = np.zeros_like(got)
    for i, t in enumerate(ts):
        v = {k: np_producer.keyframe_value_at(tracks[k], float(t)) for k in tracks}
        ref = make_cp(lens=lens, digital=digital, video_rotation=v["VideoRotation"], params=dict(lens_correction_amount=v["LensCorrectionStrength"], light_refraction_coefficient=v["LightRefractionCoeff"]))
        ref.c.adaptive_zoom_center_offset[0] = v["ZoomingCenterX"]; ref.c.adaptive_zoom_center_offset[1] = v["ZoomingCenterY"]
        ref.c.lens_correction_amount = v["LensCorrectionStrength"]; ref.c.light_refraction_coefficient = v["LightRefractionCoeff"]
        want[i] = oracle_lib.find_fovs(ref, lens, digital, [float(t)])[0]
        if i == 7:
            rd = g.DeviceGyro(ref); want_pts = rd.undistort_points(lens, digital, pts, float(t)); rd.close()
            assert np.array_equal(got_pts, want_pts)
    assert np.allclose(got, want, rtol=1e-6, atol=0), float(np.abs(got / want - 1).max())
    assert (got == want).mean() > 0.9 and np.ptp(want) > 0.01


@pytest.mark.parametrize("kw", [dict(), dict(ow=1280, oh=720), dict(video_rotation=12.0), dict(frame_readout_time_ms=0.0),
                                dict(params=dict(lens_correction_amount=0.4)), dict(params=dict(lens_correction_amount=0.7, light_refraction_coefficient=1.33)),
                                dict(horizontal=True, inverted=True),
                                dict(lens="sony"), dict(lens="opencv_standard", digital="digital_stretch"), dict(lens="gopro", digital="gopro_warp"),
                                dict(digital="gopro_superview", params=dict(lens_correction_amount=0.4)), dict(lens="poly5", params=dict(lens_correction_amount=0.7)),
                                dict(lens="insta360"), dict(lens="generic_polynomial", digital="gopro_hyperview")])
def test_oracle_find_fov_matches_second_restatement(kw):
    """FovIterative::find_fov over undistort_points_with_rolling_shutter, restated a second time in numpy scalars (tests/np_zoom.py, from
    fov_iterative.rs:76-200, cpu_undistort.rs:652-858, frame_transform.rs:352-410) == the C oracle, bit for bit: numpy's f64 slerp and
    matrix products round like the oracle's on the host."""
    import warnings
    from tests import np_zoom
    kw = dict(kw); lens = kw.pop("lens", "opencv_fisheye"); digital = kw.pop("digital", None)
    cp = make_cp(lens=lens, digital=digital, **dict(kw))
    ts = np.arange(0, 120, 17) * (1000.0 / 60.0)
    want = oracle_lib.find_fovs(cp, lens, digital, ts)
    org = (cp.c.output_width, cp.c.output_height)
    adj = make_cp(lens=lens, digital=digital, **dict(kw))             # calculate_fovs adjustments, zooming/mod.rs:41-49
    adj.c.fov_scale = 1.0; adj.c.n_fovs = 0; adj.c.n_minimal_fovs = 0; adj.c.output_width = adj.c.width; adj.c.output_height = adj.c.height
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = np.array([np_zoom.find_fov(adj, org, float(t), i, lens=lens, digital=digital) for i, t in enumerate(ts)])
    assert np.array_equal(got, want), (got, want)
    assert 0.3 < want.min() and want.max() < 3.0


def _zoom_stab(frames, h, seed=5):
    rng = np.random.default_rng(seed)
    out = []
    for f in range(frames):
        pos = np.linspace(200.0, 3800.0, 9)
        ibis = np.stack([9.0e4 * np.sin(pos / 500.0 + f), 7.0e4 * np.cos(pos / 700.0 + 0.3 * f), 900.0 * np.sin(pos / 900.0 + f)], axis=1) + rng.normal(0, 500.0, (9, 3))
        ois = np.stack([6.0e4 * np.cos(pos / 300.0 + f), 4.0e4 * np.sin(pos / 450.0), np.zeros_like(pos)], axis=1)
        out.append(dict(offset=12.5, sensor_size=(6000, 4000), crop_area=(500.0, 300.0, 5000.0, 3400.0), pixel_pitch=(8400, 8400), ibis=(pos, ibis), ois=(pos, ois)))
    return out


@pytest.mark.parametrize("kw", [dict(), dict(frame_readout_time_ms=0.0), dict(lens="sony", params=dict(lens_correction_amount=0.6)),
                                dict(frame_readout_time_ms=0.0, suppress=True)])
def test_point_path_ibis_shifts_oracle_matches_second_restatement(kw):
    """The IBIS / OIS `shifts` of at_timestamp_for_points (frame_transform.rs:412-434) and their use in undistort_points
    (cpu_undistort.rs:748-757, where y is rotated with the already rotated x): C oracle == tests/np_zoom.py.  With rolling-shutter
    correction off only the FIRST point is shifted (points_iter is the single point (0, 0)); with suppress_rotation on top, none."""
    import warnings
    from tests import np_zoom
    kw = dict(kw); lens = kw.pop("lens", "opencv_fisheye"); suppress = kw.pop("suppress", False)
    stab = _zoom_stab(3, 1080)
    cp = make_cp(lens=lens, camera_stab=stab, **kw)
    plain = make_cp(lens=lens, **kw)
    if suppress: cp.c.suppress_rotation = 1; plain.c.suppress_rotation = 1
    lib = oracle_lib.load()
    pts = np.array([[3.0, 2.0], [960.0, 540.0], [1900.0, 30.0], [40.0, 1070.0], [1500.0, 800.0]], np.float32)
    for frame, ts in enumerate((300.0, 1500.0, 2900.0)):
        lca = float(cp.c.lens_correction_amount)
        want = np.zeros_like(pts); base = np.zeros_like(pts)
        lib.gf_oracle_undistort_points_rs_ex(C.byref(cp.c), abi.LENS[lens], 0, pts.ctypes.data, len(pts), ts, frame, lca, 0, want.ctypes.data)
        lib.gf_oracle_undistort_points_rs_ex(C.byref(plain.c), abi.LENS[lens], 0, pts.ctypes.data, len(pts), ts, frame, lca, 0, base.ctypes.data)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            got = np.array(np_zoom.undistort_points_with_rolling_shutter(cp, [tuple(p) for p in pts], ts, frame, lca, False, lens, None, stab[frame]), np.float32)
        assert np.array_equal(got, want), (got, want)
        moved = np.abs(want - base).max(axis=1) > 0.5
        if suppress:                      assert not moved.any()
        elif "frame_readout_time_ms" in kw: assert moved[0] and not moved[1:].any()
        else:                             assert moved.all()


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(frame_readout_time_ms=0.0), dict(lens="sony", params=dict(lens_correction_amount=0.6))])
def test_device_point_path_with_ibis_shifts_matches_oracle(kw):
    """The zoom kernels apply the per-point IBIS / OIS shifts (frame_transform.rs:412-434, cpu_undistort.rs:748-757) from the spline points in
    HBM: undistort_points and find_fovs on the device == the oracle (which test_point_path_ibis_shifts_oracle_matches_second_restatement
    ties to the second transcription), including the rolling-shutter-off quirk (only the first point of a call is shifted)."""
    kw = dict(kw); lens = kw.pop("lens", "opencv_fisheye")
    n = 24
    stab = _zoom_stab(n, 1080)
    cp = make_cp(lens=lens, camera_stab=stab, **kw)
    lib = oracle_lib.load()
    dg = g.DeviceGyro(cp)
    pts = np.array([[3.0, 2.0], [960.0, 540.0], [1900.0, 30.0], [40.0, 1070.0], [1500.0, 800.0]], np.float32)
    lca = float(cp.c.lens_correction_amount)
    for frame, ts in ((0, 300.0), (7, 1500.0), (20, 2900.0)):
        want = np.zeros_like(pts)
        lib.gf_oracle_undistort_points_rs_ex(C.byref(cp.c), abi.LENS[lens], 0, pts.ctypes.data, len(pts), ts, frame, lca, 0, want.ctypes.data)
        got = dg.undistort_points(lens, None, pts, ts, frame=frame, lens_correction_amount=lca)
        assert np.allclose(got, want, rtol=0, atol=2e-3), (frame, got, want)
    ts = np.arange(n) * (1000.0 / 60.0) * 5
    want = oracle_lib.find_fovs(cp, lens, None, ts)
    got = dg.find_fovs(lens, None, ts)
    plain = make_cp(lens=lens, **kw)
    base = oracle_lib.find_fovs(plain, lens, None, ts)
    dg.close()
    assert np.allclose(got, want, rtol=1e-6, atol=0), float(np.abs(got / want - 1).max())
    assert np.abs(want / base - 1).max() > 1e-3          # the shifts do move the polygon


def _distorting_mesh(w, h, fpd, rows=9):
    from gyroflow_b200 import synth
    return np.asarray(synth.synthetic_mesh(w, h, amp=6.0, n=rows, with_fpd=fpd), dtype=np.float64)     # same layout as mesh_correction[frame].0 (sony.rs:483-511)


@pytest.mark.parametrize("fpd", [False, True])
def test_point_path_distorting_mesh_oracle_matches_second_restatement(fpd):
    """The mesh block of undistort_points (cpu_undistort.rs:712-746: focal-plane distortion ADDED, then the distorting mesh through the f64
    bivariate spline): C oracle == tests/np_zoom.py, with and without the focal-plane block, combined with IBIS shifts."""
    import warnings
    from tests import np_zoom
    stab = _zoom_stab(2, 1080)
    meshes = [_distorting_mesh(1920, 1080, fpd), None]
    cp = make_cp(lens="sony", camera_stab=stab, distorting_meshes=meshes)
    plain = make_cp(lens="sony", camera_stab=stab)
    lib = oracle_lib.load()
    pts = np.array([[3.0, 2.0], [960.0, 540.0], [1900.0, 30.0], [40.0, 1070.0], [1500.0, 800.0]], np.float32)
    for frame, ts in enumerate((300.0, 1500.0)):
        want = np.zeros_like(pts); base = np.zeros_like(pts)
        lib.gf_oracle_undistort_points_rs_ex(C.byref(cp.c), abi.LENS["sony"], 0, pts.ctypes.data, len(pts), ts, frame, 1.0, 0, want.ctypes.data)
        lib.gf_oracle_undistort_points_rs_ex(C.byref(plain.c), abi.LENS["sony"], 0, pts.ctypes.data, len(pts), ts, frame, 1.0, 0, base.ctypes.data)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            mesh = None if meshes[frame] is None else [float(v) for v in meshes[frame]]
            got = np.array(np_zoom.undistort_points_with_rolling_shutter(cp, [tuple(p) for p in pts], ts, frame, 1.0, False, "sony", None, stab[frame], mesh), np.float32)
        assert np.array_equal(got, want), (got, want)
        assert (np.abs(want - base).max() > 1.0) == (frame == 0)          # frame 1 has no mesh


@pytest.mark.gpu
@pytest.mark.parametrize("fpd,rows", [(False, 9), (True, 9), (False, 7), (True, 7)], ids=["False", "True", "False-7rows", "True-7rows"])
def test_device_point_path_with_distorting_mesh_matches_oracle(fpd, rows):
    """9-row meshes take the unrolled spline (mesh_interpolate9), other grids the general one (mesh_bivariate)."""
    n = 12
    meshes = [_distorting_mesh(1920, 1080, fpd, rows) if i % 3 != 2 else None for i in range(n)]
    cp = make_cp(lens="sony", camera_stab=_zoom_stab(n, 1080), distorting_meshes=meshes)
    lib = oracle_lib.load()
    dg = g.DeviceGyro(cp)
    pts = np.array([[3.0, 2.0], [960.0, 540.0], [1900.0, 30.0], [40.0, 1070.0], [1500.0, 800.0]], np.float32)
    for frame, ts in ((0, 300.0), (2, 900.0), (7, 1500.0)):
        want = np.zeros_like(pts)
        lib.gf_oracle_undistort_points_rs_ex(C.byref(cp.c), abi.LENS["sony"], 0, pts.ctypes.data, len(pts), ts, frame, 1.0, 0, want.ctypes.data)
        got = dg.undistort_points("sony", None, pts, ts, frame=frame)
        assert np.allclose(got, want, rtol=0, atol=2e-3), (frame, got, want)
    ts = np.arange(n) * (1000.0 / 60.0) * 9
    want = oracle_lib.find_fovs(cp, "sony", None, ts)
    got = dg.find_fovs("sony", None, ts)
    dg.close()
    assert np.allclose(got, want, rtol=1e-6, atol=0), float(np.abs(got / want - 1).max())
