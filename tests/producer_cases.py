"""One table of producer configurations (FrameTransform::at_timestamp, frame_transform.rs:165-350), shared by the CPU test of the host
producer against the numpy restatement (tests/np_producer.py) and the GPU tests of the device producer against the host producer.

Each case: ComputeParams keyword arguments (`kw`), direct gf_compute_params overrides (`c`), a frame size and (timestamp, frame) pairs.
`null` lists (frame, spline name) pairs whose camera_stab pointers are set to null after construction, with the point count kept."""
import ctypes as C

import numpy as np

import gyroflow_b200 as g
from gyroflow_b200 import synth
from tests import cases, np_producer

BLOCK = 128                                  # rows per block of frame_rows_kernel
SENSOR, CROP, PITCH, OFFSET = (6000, 4000), (500.0, 300.0, 5000.0, 3400.0), (8400, 8400), 12.5


def ulp_diff(a, b):
    a = np.asarray(a, np.float32); b = np.asarray(b, np.float32)
    return np.abs(a - b) / np.maximum(np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32)), np.float32(1e-45))


def table_ulp_max(m, want):
    """Largest f32 ulp distance of a producer table's columns 0-8 from the numpy restatement.  A difference below one f64 ulp of the
    row's largest entry counts as none: that is rounding noise of either inverse (numpy's SVD pinv leaves ~1e-19 where the cofactor
    inverse has 0, and entries near 1e-10 come out of cancellation), not a difference of the producers."""
    m = np.asarray(m, np.float32); want = np.asarray(want, np.float32)
    u = ulp_diff(m, want)
    scale = np.abs(want.astype(np.float64)).max(axis=1, keepdims=True)
    u[np.abs(m.astype(np.float64) - want) <= scale * 2.0 ** -52] = 0.0
    return float(u.max())


def spline_stab(counts, seed=3, ois=True, band=None):
    """CameraStabData per frame (sensor 6000 x 4000, crop (500, 300, 5000, 3400), 8.4 um pitch).  counts[f] spline points for frame
    f — a count of 0 gives an entry without splines.  band: (lo, hi) spline-position range (sensor rows + offset) per frame, or None
    for the whole crop."""
    rng = np.random.default_rng(seed)
    out = []
    for f, n in enumerate(counts):
        d = dict(offset=OFFSET, sensor_size=SENSOR, crop_area=CROP, pixel_pitch=PITCH)
        if n:
            lo, hi = band[f] if band else (250.0, 3750.0)
            pos = np.linspace(lo, hi, n)
            if not band:
                pos = np.sort(pos + rng.uniform(-10.0, 10.0, n))
            ibis = np.stack([2.0e5 * np.sin(pos / 700.0 + f) + 3.0e4, -1.5e5 * np.cos(pos / 500.0) + 2.0e4, 150.0 * np.sin(pos / 900.0 + 0.3 * f) + 40.0], axis=1)
            d["ibis"] = (pos, ibis)
            if ois:
                d["ois"] = (pos, np.stack([6.0e4 * np.cos(pos / 300.0 + f), 4.0e4 * np.sin(pos / 450.0) + 1.0e4, np.zeros_like(pos)], axis=1))
        out.append(d)
    return out


def band_for_rows(h, r0, r1):
    """Spline-position range whose Catmull-Rom span covers frame rows r0 .. r1 - 1 of an h-row frame (no framebuffer inversion)."""
    ys = lambda y: y * (CROP[3] / h) + CROP[1] + OFFSET         # map_coord + offset, frame_transform.rs:270-275
    return ys(r0), ys(r1 - 1)


def _lens(n):
    out = []
    for i in range(n):
        K = [480.0 * (1.0 + 0.1 * i), 0.0, 320.0 + 3.0 * i, 0.0, 470.0 * (1.0 + 0.07 * i), 180.0 - 2.0 * i, 0.0, 0.0, 1.0]
        out.append(dict(camera_matrix=K, distortion_coeffs=[0.05 * (1 - 0.2 * i), 0.01, -0.002, 0.0005] + [0.0] * 8, radial_distortion_limit=0.5 * i,
                        input_horizontal_stretch=1.0 + 0.25 * i, input_vertical_stretch=1.0 - 0.1 * i))
    return out


TS3 = [(250.0, 0), (1234.5, 1), (3100.0, 2)]
SYNC3 = {1_000_000: 2.0, 1_800_000: -3.0, 2_600_000: 5.0}
VARYING = [24, 7, 40, 12, 3]                                  # spline points per frame: frame 0's count is wrong for every other frame
STAB_TS = [(400.0, 0), (1200.0, 1), (2300.0, 2), (2950.0, 3), (3500.0, 4), (3700.0, 5), (3950.0, 9)]   # frames 5, 9: past the end

CASES = {
    "default":            dict(frames=TS3),
    "horizontal":         dict(kw=dict(horizontal=True), frames=TS3),
    "readout_inverted":   dict(kw=dict(frame_readout_time_ms=9.5, inverted=True), frames=TS3),
    "fb_inverted":        dict(kw=dict(framebuffer_inverted=True), frames=TS3),
    "fb_inverted_horizontal": dict(kw=dict(framebuffer_inverted=True, horizontal=True), frames=TS3),
    "readout_zero":       dict(kw=dict(frame_readout_time_ms=0.0), frames=TS3),
    "readout_zero_stab":  dict(kw=dict(frame_readout_time_ms=0.0, camera_stab=spline_stab(VARYING)), frames=STAB_TS),
    "readout_time_scale": dict(kw=dict(readout_time_scale=0.85), frames=TS3),
    "video_rotation":     dict(kw=dict(video_rotation=17.0), frames=TS3),
    "suppress_rotation_rs": dict(kw=dict(camera_stab=spline_stab(VARYING)), c=dict(suppress_rotation=1), frames=STAB_TS),
    "suppress_rotation_no_rs": dict(kw=dict(frame_readout_time_ms=0.0, camera_stab=spline_stab(VARYING)), c=dict(suppress_rotation=1), frames=STAB_TS),
    "lens_per_frame":     dict(kw=dict(lens_per_frame=_lens(2)), frames=[(300.0, 0), (1500.0, 1), (2900.0, 2)]),
    "focal_lengths":      dict(kw=dict(focal_lengths=[24.0, float("nan"), 26.0], smoothed_focal_lengths=[24.2, 25.0, 25.5]),
                               frames=[(300.0, 0), (1500.0, 1), (2900.0, 2), (3600.0, 3)]),
    "gyro_offset_scalar": dict(kw=dict(gyro_offset_ms=6.5), frames=TS3),
    "one_sync_point":     dict(kw=dict(sync_offsets={1_500_000: -4.0}, gyro_offset_ms=3.0), frames=TS3),
    "sync_points":        dict(kw=dict(sync_offsets=SYNC3), frames=[(100.0, 0), (1400.0, 1), (2200.0, 2), (3900.0, 3)]),
    "per_frame_time_offsets": dict(kw=dict(per_frame_time_offsets=[0.0, -4.0, 2.5]), frames=[(300.0, 0), (1500.0, 1), (2900.0, 2), (3600.0, 3)]),
    "stab_varying":       dict(kw=dict(camera_stab=spline_stab(VARYING), sync_offsets=SYNC3, per_frame_time_offsets=[0.25 * i for i in range(6)],
                                       readout_time_scale=0.9), frames=STAB_TS),
    "stab_ibis_only":     dict(kw=dict(camera_stab=spline_stab(VARYING[::-1], seed=4, ois=False)), frames=STAB_TS),
    "stab_fb_inverted":   dict(kw=dict(camera_stab=spline_stab(VARYING, seed=6), framebuffer_inverted=True), frames=STAB_TS),
    "stab_band":          dict(kw=dict(camera_stab=spline_stab([9, 16], band=[band_for_rows(360, 40, 90), band_for_rows(360, 200, 330)])),
                               frames=[(700.0, 0), (1700.0, 1), (2700.0, 2)]),
    "stab_null_pointers": dict(kw=dict(camera_stab=spline_stab(VARYING)), null=[(0, "ibis"), (1, "ois"), (2, "ibis"), (2, "ois")], frames=STAB_TS),
    "tall":               dict(w=1024, h=4320, kw=dict(camera_stab=spline_stab([30, 11]), sync_offsets=SYNC3),
                               frames=[(600.0, 0), (2100.0, 1), (3300.0, 2)]),
    "wide_horizontal":    dict(w=3840, h=2160, kw=dict(horizontal=True, camera_stab=spline_stab([14, 33]), gyro_offset_ms=-2.0),
                               frames=[(800.0, 0), (2500.0, 1), (3800.0, 4)]),
}


def make(case, org=None, sm=None):
    """(KernelParams, ComputeParams, camera_stab as the producer sees it) for one case."""
    w, h = case.get("w", 640), case.get("h", 360)
    p = synth.base_kernel_params(w, h)
    if org is None:
        org, sm = cases.gyro()
    kw = case.get("kw", {})
    cp = g.ComputeParams(p, org, sm, **kw)
    for name, v in case.get("c", {}).items():
        setattr(cp.c, name, v)
    stab = kw.get("camera_stab")
    if case.get("null"):
        stab = [dict(d) for d in stab]
        for f, name in case["null"]:
            setattr(cp._stab[f], name + "_pos", C.POINTER(C.c_double)())
            if name == "ois":
                setattr(cp._stab[f], name + "_xyz", C.POINTER(C.c_double)())
            assert getattr(cp._stab[f], "n_" + name) > 0          # the count stays: only the pointers say "no points"
            stab[f].pop(name)
    return p, cp, stab


def np_expected(case, p, org, sm, stab, ts, frame):
    """The numpy restatement's table for (ts, frame) of a case, and the f64 fov the producer narrows into KernelParams.fov."""
    kw = case.get("kw", {})
    frt = abs(kw.get("frame_readout_time_ms", 16.0))                    # get_frame_readout_time (:22-36)
    if kw.get("framebuffer_inverted") and not kw.get("horizontal"):
        frt = -frt
    if kw.get("inverted"):
        frt = -frt
    frt *= kw.get("readout_time_scale", 0.0) or 1.0
    pfo = kw.get("per_frame_time_offsets")
    if pfo is not None and frame < len(pfo):
        ts += pfo[frame]                                                # :224
    fl, sfl = kw.get("focal_lengths"), kw.get("smoothed_focal_lengths")
    comp = fl[frame] / sfl[frame] if fl is not None and frame < len(fl) and fl[frame] > 0 and sfl[frame] > 0 else 1.0   # :70-80
    fov = max(kw.get("fov_scale", 1.0), 0.001) * (p.width / p.output_width) * comp                                     # get_fov :52-58
    lens = kw.get("lens_per_frame")
    K = lens[frame]["camera_matrix"] if lens and frame < len(lens) else None
    m = np_producer.frame_matrices(p, org, sm, ts, frame_readout_time_ms=frt, video_rotation_deg=kw.get("video_rotation", 0.0),
                                   horizontal=kw.get("horizontal", False), framebuffer_inverted=kw.get("framebuffer_inverted", False),
                                   offsets=kw.get("sync_offsets"), gyro_offset_ms=kw.get("gyro_offset_ms", 0.0),
                                   suppress_rotation=bool(case.get("c", {}).get("suppress_rotation")), camera_stab=stab, frame=frame,
                                   camera_matrix=K, fov_f64=fov)
    return m, fov


def compare_tables(dev, host):
    """The device producer's table against the host producer's: columns 9-13 (IBIS / OIS: plain f64 + - * / with contraction off on
    both sides) bit-identical, columns 0-8 within 1 f32 ulp (device acos / sin in qslerp).  Returns the bit-identical count of 0-8."""
    assert dev.shape == host.shape
    bad = np.nonzero(dev[:, 9:].view(np.uint32) != host[:, 9:].view(np.uint32))
    assert bad[0].size == 0, "IBIS / OIS columns differ at rows %s" % sorted(set(bad[0].tolist()))[:8]
    u = ulp_diff(dev[:, :9], host[:, :9])
    STATS["max_ulp"] = max(STATS["max_ulp"], float(u.max()))
    assert float(u.max()) <= 1.0, "columns 0-8: %.1f ulp at row %d" % (float(u.max()), int(np.argmax(u.max(axis=1))))
    return int((dev[:, :9].view(np.uint32) == host[:, :9].view(np.uint32)).sum())


STATS = dict(max_ulp=0.0)                      # largest columns 0-8 difference compare_tables saw, for the report


def table_flags_host(table):
    t = np.ascontiguousarray(table, dtype=np.float32)
    return int(g.load_library().gf_table_flags_host(t.ctypes.data, t.shape[0]))
