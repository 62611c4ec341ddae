"""The adaptive-zoom point path (zoom_kernel.cu) against the CPU oracle, cell by cell.

A cell is one (lens pair, option row).  The pairs are every (lens, digital lens) the point path compiles: the 21 the reference
pre-compiles plus (gopro, digital_stretch), since pick_digital takes digital_stretch for every model.  The option rows are the
settings that change the arithmetic of undistort_points: lens-correction strength, refraction, input stretch, output size and zoom
centre, readout direction, IBIS / OIS shifts, distorting meshes with and without focal-plane data, keyframed values, use_fovs, the
lens_noop branch, frame sizes, and a few extreme rows for particular pairs.

With suppress_rotation set no f64 libm result reaches the output: the rotation is the identity and K_new is plain arithmetic, and
everything after it is f32 code shared with the warp.  So the rotation-free cells compare bit for bit (two NaNs count as equal,
whatever their payload: the host's default NaN is not the GPU's).  Each runs undistort_points, find_fovs, stmap_distort_dev,
generate_stmap (per_frame on and off) and, where the oracle takes the row's inputs, calculate_fovs.  The cells are counted, so that
none drops out silently; the report lists every failing cell and the test fails on the first difference.

The rotation-on cells (one per pair, with rolling shutter and IBIS on) keep the bars of the rotation's f64 slerp: its acos / sin
differ by an ulp between the device and glibc.

test_oracle_matches_second_restatement ties the oracle to tests/np_zoom.py over the same pairs and rows, without a GPU.
"""
import ctypes as C
import time
import warnings

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi
from tests import np_producer, oracle_lib
from tests.test_kernel_matrix import REFERENCE_PAIRS, report
from tests.test_zoom import _distorting_mesh, _zoom_stab, make_cp

POINT_PAIRS = REFERENCE_PAIRS + [("gopro", "digital_stretch")]
GF_ERR_UNSUPPORTED_COMBO = -5        # include/gyroflow_cuda.h
DURATION_MS = 4000.0                # cases.gyro(): samples from 0 to 4 s
# before the first gyro sample, inside, repeated, after the clip's duration
FOV_TS = [-50.0, 1234.5, 1234.5, DURATION_MS + 100.0]
POINT_COUNTS = (1, 127, 128, 129, 4097)
STMAP_SIZE = (67, 41)               # w * h is not a multiple of the 128-thread block
SENTINEL = 0x7FA5A5A5               # a NaN no kernel writes


# ---- points ----------------------------------------------------------------------------------------------------------------------
def point_set(w, h, n=4097):
    """n points: value edges first (so that the short counts hold them), then the principal point and the axes through it, the
    corners and edge midpoints, far off-axis points, and a grid over [-0.25w, 1.25w] x [-0.25h, 1.25h]."""
    cx, cy = w / 2.0, h / 2.0                        # synth.base_kernel_params: the principal point is the frame centre
    nan, inf = float("nan"), float("inf")
    pts = [(cx, cy), (nan, cy), (cx, nan), (nan, nan), (inf, cy), (-inf, cy), (cx, inf), (cx, -inf), (inf, -inf),
           (1e30, cy), (-1e30, cy), (cx, 1e30), (1e30, -1e30), (-0.0, -0.0), (-0.0, cy), (cx, -0.0)]
    pts += [(cx + d, cy) for d in np.linspace(-0.75 * w, 0.75 * w, 13)] + [(cx, cy + d) for d in np.linspace(-0.75 * h, 0.75 * h, 13)]
    pts += [(0, 0), (w, 0), (0, h), (w, h), (w - 1, h - 1), (cx, 0), (cx, h), (0, cy), (w, cy)]
    pts += [(40.0 * w, 30.0 * h), (-20.0 * w, 5.0 * h), (200.0 * w, cy), (cx, -60.0 * h), (3.0 * w, 2.5 * h)]
    m = n - len(pts)
    nx = int(np.ceil(np.sqrt(m * w / h)))
    ny = -(-m // nx)
    gx, gy = np.meshgrid(np.linspace(-0.25 * w, 1.25 * w, nx), np.linspace(-0.25 * h, 1.25 * h, ny))
    pts += list(zip(gx.ravel()[:m], gy.ravel()[:m]))
    return np.asarray(pts, np.float32)


def same_bits(a, b):
    """Elementwise: identical bits, or both NaN."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.shape != b.shape:
        return np.zeros(1, bool)
    u = {4: np.uint32, 8: np.uint64}[a.dtype.itemsize]
    return (a.view(u) == b.view(u)) | (np.isnan(a) & np.isnan(b))


def first_diff(got, want):
    ok = same_bits(got, want)
    if ok.size == 1 and got.size != 1:
        return "shape %s != %s" % (got.shape, want.shape)
    i = int(np.flatnonzero(~ok.ravel())[0])
    return "%d of %d values differ, first at %d: got %r want %r" % (int((~ok).sum()), ok.size, i, got.ravel()[i], want.ravel()[i])


# ---- option rows -----------------------------------------------------------------------------------------------------------------
def _meshes(rows, fpd):
    # frame 0 and 2 have a mesh, frame 1 has none; frames >= 3 are past the end of the mesh and stab arrays
    return lambda w, h: dict(distorting_meshes=[_distorting_mesh(w, h, fpd, rows), None, _distorting_mesh(w, h, fpd, rows)],
                             camera_stab=_zoom_stab(3, h))


KEYS = {"ZoomingCenterX": [(100_000, -0.04, "EaseIn"), (1_500_000, 0.05, "EaseInOut")],
        "ZoomingCenterY": [(0, 0.03, "NoEasing"), (1_900_000, -0.02, "EaseOut")],
        "LensCorrectionStrength": [(0, 1.0, "EaseInOut"), (1_000_000, 0.35, "EaseInOut"), (2_000_000, 0.8, "EaseIn")],
        "LightRefractionCoeff": [(0, 1.0, "NoEasing"), (2_000_000, 1.33, "NoEasing")]}
FOV_KEYS = {"Fov": [(0, 0.8, "EaseIn"), (1_500_000, 1.6, "EaseOut"), (3_000_000, 1.1, "NoEasing")]}
# (frame, timestamp) of the undistort_points / stmap_distort_dev calls
FRAMES = [(0, 1234.5)]
MESH_FRAMES = [(0, 300.0), (1, 1500.0), (2, 2100.0), (5, 2900.0)]
KEYED_FRAMES = [(0, 200.0), (3, 1300.0), (7, 2600.0)]


def row(name, kw=None, c=None, **extra):
    """An option row.  kw(w, h): make_cp arguments; c: gf_compute_params fields set afterwards; extra: margins, frames, fov_ts,
    use_fovs, keyed (the row has keyframes, so the oracle runs on constants), pairs (restrict to these pairs), calc (run
    calculate_fovs), size (w, h of the main cp), np_zoom (the second transcription covers the row), stmap (run the ST-map entry
    points on a STMAP_SIZE frame), counts (also run POINT_COUNTS), sentinel (the Newton solve must give up somewhere)."""
    r = dict(name=name, kw=kw or (lambda w, h: {}), c=c or {}, margins=(2.0,), frames=FRAMES, fov_ts=FOV_TS, use_fovs=False, keyed=False,
             pairs=None, calc=True, size=(1920, 1080), np_zoom=True, stmap=True)
    r.update(extra)
    return r


ZERO_K = dict(distortion_coeffs=[0.0] * 12)
ROWS = [
    row("plain", fov_ts=FOV_TS + list(np.arange(0, 257 - len(FOV_TS)) * (1000.0 / 60.0)), counts=True),
    row("lc0.4", lambda w, h: dict(params=dict(lens_correction_amount=0.4))),
    row("lc0.0", lambda w, h: dict(params=dict(lens_correction_amount=0.0))),         # the factor is clamped to 0.001
    row("lc0.7-refraction1.33", lambda w, h: dict(params=dict(lens_correction_amount=0.7, light_refraction_coefficient=1.33))),
    row("stretch1.25x0.9", c=dict(input_horizontal_stretch=1.25, input_vertical_stretch=0.9)),
    row("stretch0.001", c=dict(input_horizontal_stretch=0.001, input_vertical_stretch=0.001)),      # not applied (> 0.001 is)
    row("out1280x720-centre-margins", lambda w, h: dict(ow=w * 2 // 3, oh=h * 2 // 3), c=dict(adaptive_zoom_center_offset=[0.03, -0.02]),
        margins=(0.0, 2.0, 37.5)),
    row("horizontal", lambda w, h: dict(horizontal=True)),
    row("ibis-rs", lambda w, h: dict(camera_stab=_zoom_stab(3, h)), frames=[(0, 300.0), (2, 2900.0), (4, 1000.0)]),
    # rotation suppressed and readout off: no shifts at all (frame_transform.rs:432-434)
    row("ibis-readout-off", lambda w, h: dict(camera_stab=_zoom_stab(3, h), frame_readout_time_ms=0.0), frames=[(0, 300.0), (2, 2900.0)]),
    row("mesh9", _meshes(9, False), frames=MESH_FRAMES),
    row("mesh9-fpd", _meshes(9, True), frames=MESH_FRAMES),
    row("mesh7", _meshes(7, False), frames=MESH_FRAMES),
    row("mesh7-fpd", _meshes(7, True), frames=MESH_FRAMES),
    row("keyframes", lambda w, h: dict(keyframes=KEYS), frames=KEYED_FRAMES, fov_ts=[200.0, 1300.0, 2600.0, 1300.0], keyed=True, np_zoom=False),
    row("use-fovs-array", lambda w, h: dict(fovs=[0.7, 1.3, 2.2]), frames=[(0, 100.0), (2, 900.0), (6, 1500.0)], use_fovs=True),
    row("use-fovs-track", lambda w, h: dict(fovs=[0.9, 1.2], keyframes=FOV_KEYS), frames=KEYED_FRAMES, use_fovs=True, keyed=True, np_zoom=False),
    row("zero-coefficients", c=ZERO_K),                                                # lens_noop for fisheye, sony, generic polynomial, gopro
    row("portrait1080x1920", size=(1080, 1920)),
    row("small16x12", size=(16, 12)),
    row("8k7680x4320", size=(7680, 4320), stmap=False),
    # extreme rows for particular pairs
    row("gopro-past-89deg", lambda w, h: dict(fovs=[3.0], params=dict(lens_correction_amount=0.5)), use_fovs=True,
        pairs=[("gopro", None), ("gopro", "gopro_warp"), ("gopro", "digital_stretch")]),
    row("poly3-newton-gives-up", c=dict(distortion_coeffs=[0.3] + [0.0] * 11), pairs=[("poly3", None), ("poly3", "digital_stretch")], sentinel=True),
    row("digital-fixed-point-diverges", lambda w, h: dict(params=dict(lens_correction_amount=0.3)), c=dict(distortion_coeffs=[0.4, 0.2, 0.05, 0.01] + [0.0] * 8),
        pairs=[("opencv_fisheye", d) for d in ("gopro_superview", "gopro6_superview", "gopro_hyperview")]),
]


def row_pairs(r):
    return r["pairs"] or POINT_PAIRS


def build_cp(r, lens, digital, w, h, suppress=True, constants_at=None):
    """The row's ComputeParams at w x h.  constants_at: a timestamp — the keyframed values at it become constants (the oracle's view)."""
    kw = dict(r["kw"](w, h))
    keys = kw.pop("keyframes", None)
    if keys and constants_at is None:
        kw["keyframes"] = keys
    cp = make_cp(w=w, h=h, lens=lens, digital=digital, **kw)
    for k, v in r["c"].items():
        if isinstance(v, list):
            getattr(cp.c, k)[:] = v
        else:
            setattr(cp.c, k, v)
    if keys and constants_at is not None:
        val = {k: np_producer.keyframe_value_at(keys[k], float(constants_at)) for k in keys}
        if "ZoomingCenterX" in val: cp.c.adaptive_zoom_center_offset[0] = val["ZoomingCenterX"]
        if "ZoomingCenterY" in val: cp.c.adaptive_zoom_center_offset[1] = val["ZoomingCenterY"]
        if "LensCorrectionStrength" in val: cp.c.lens_correction_amount = val["LensCorrectionStrength"]
        if "LightRefractionCoeff" in val: cp.c.light_refraction_coefficient = val["LightRefractionCoeff"]
        if "Fov" in val: cp.c.fov_scale = val["Fov"]
    cp.c.suppress_rotation = int(suppress)
    return cp


def oracle_points(cp, lens, digital, pts, ts, frame, lca, use_fovs):
    out = np.zeros_like(pts)
    oracle_lib.load().gf_oracle_undistort_points_rs_ex(C.byref(cp.c), abi.LENS[lens], abi.LENS[digital] if digital else 0, pts.ctypes.data, len(pts),
                                                        ts, frame, lca, int(use_fovs), out.ctypes.data)
    return out


def oracle_stmap_distort(cp, lens, digital, ts, frame):
    out = np.zeros((cp.c.height, cp.c.width, 3), np.float32)
    oracle_lib.load().gf_oracle_stmap_distort(C.byref(cp.c), abi.LENS[lens], abi.LENS[digital] if digital else 0, ts, frame, out.ctypes.data)
    return out


def device_stmap_distort(dg, lens, digital, ts, frame):
    """gf_cuda_stmap_distort_dev on a side stream into a buffer pre-filled with SENTINEL past the map: returns (map, tail intact)."""
    import torch
    n = dg.cp.c.width * dg.cp.c.height * 3
    buf = torch.full((n + 1024,), SENTINEL, dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    rc = dg._lib.gf_cuda_stmap_distort_dev(dg._h, C.byref(dg.cp.c), abi.LENS[lens], abi.LENS[digital] if digital else 0, ts, frame,
                                           buf.data_ptr(), side.cuda_stream)
    if rc != 0:
        raise g.GyroflowCoreError(rc, "gf_cuda_stmap_distort_dev")
    side.synchronize()
    host = buf.cpu().numpy()
    return host[:n].view(np.float32).reshape(dg.cp.c.height, dg.cp.c.width, 3), bool((host[n:] == SENTINEL).all())


# ---- the matrix ------------------------------------------------------------------------------------------------------------------
class Tally:
    def __init__(self):
        self.cells, self.checks, self.bad, self.bad_cells = set(), 0, [], set()

    def check(self, cell, what, got, want):
        self.checks += 1
        ok = same_bits(got, want)
        if not ok.all():
            self.bad.append("%s %s: %s" % (cell, what, first_diff(np.asarray(got), np.asarray(want))))
            self.bad_cells.add(cell)

    def require(self, cell, what, cond):
        self.checks += 1
        if not cond:
            self.bad.append("%s %s" % (cell, what))
            self.bad_cells.add(cell)


def run_cell(t, r, lens, digital):
    """Every entry point of one rotation-free cell against the oracle."""
    from tests.test_stmap import oracle_stmap
    from tests.test_zoom_fovs import MODES, _oracle, _per_frame
    cell = (lens, digital, r["name"])
    w, h = r["size"]
    cp = build_cp(r, lens, digital, w, h)
    lca = float(cp.c.lens_correction_amount)
    pts = point_set(w, h)
    dg = g.DeviceGyro(cp)
    try:
        for frame, ts in r["frames"]:
            ref = build_cp(r, lens, digital, w, h, constants_at=ts) if r["keyed"] else cp
            want = oracle_points(ref, lens, digital, pts, ts, frame, lca, r["use_fovs"])
            got = dg.undistort_points(lens, digital, pts, ts, frame=frame, use_fovs=r["use_fovs"], lens_correction_amount=lca)
            t.check(cell, "undistort_points frame %d" % frame, got, want)
            if r.get("sentinel"):
                t.require(cell, "the Newton solve gives up somewhere (-1e6 sentinel)", (want == -1000000.0).any())
            if r.get("counts"):
                for n in POINT_COUNTS[:-1]:
                    # first n + 1 points shifted by one, so that a point the next call leaves unwritten in a reused output
                    # allocation holds its neighbour's value rather than its own
                    shifted = pts[1:n + 2]
                    got = dg.undistort_points(lens, digital, shifted, ts, frame=frame, use_fovs=r["use_fovs"], lens_correction_amount=lca)
                    t.check(cell, "undistort_points n=%d" % (n + 1), got, oracle_points(cp, lens, digital, shifted, ts, frame, lca, r["use_fovs"]))
                    got = dg.undistort_points(lens, digital, pts[:n], ts, frame=frame, use_fovs=r["use_fovs"], lens_correction_amount=lca)
                    t.check(cell, "undistort_points n=%d" % n, got, want[:n])
        for margin in r["margins"]:
            ts = np.asarray(r["fov_ts"])
            got = dg.find_fovs(lens, digital, ts, margin=margin)
            if r["keyed"]:
                want = np.array([oracle_lib.find_fovs(build_cp(r, lens, digital, w, h, constants_at=x), lens, digital, [x], margin)[0] for x in ts])
            else:
                want = oracle_lib.find_fovs(cp, lens, digital, ts, margin)
            t.check(cell, "find_fovs margin %g" % margin, got, want)
        if r["calc"] and not r["keyed"]:
            kw = dict(MODES["dynamic-gaussian"], scaled_fps=30.0, fov_algorithm_margin=r["margins"][-1])
            ts = np.asarray(r["fov_ts"])
            got, got_min = dg.calculate_fovs(lens, digital, g.ZoomParams(**kw), ts)
            window, speed, zk, sk = _per_frame(kw, ts)
            want, want_min = np.zeros(ts.size), np.zeros(ts.size)
            zp = g.ZoomParams(**kw)
            _oracle().gf_oracle_calculate_fovs(C.byref(cp.c), C.byref(zp.c), abi.LENS[lens], abi.LENS[digital] if digital else 0, ts.ctypes.data,
                                               window.ctypes.data, speed.ctypes.data, zk, sk, ts.size, want.ctypes.data, want_min.ctypes.data)
            t.check(cell, "calculate_fovs", got, want)
            t.check(cell, "calculate_fovs minimal", got_min, want_min)
    finally:
        dg.close()
    if not r["stmap"]:
        t.cells.add(cell)
        return
    sw, sh = STMAP_SIZE
    scp = build_cp(r, lens, digital, sw, sh)
    dg = g.DeviceGyro(scp)
    try:
        for frame, ts in r["frames"]:
            ref = build_cp(r, lens, digital, sw, sh, constants_at=ts) if r["keyed"] else scp
            got, tail_ok = device_stmap_distort(dg, lens, digital, ts, frame)
            t.require(cell, "stmap_distort_dev frame %d wrote past w*h*3 floats" % frame, tail_ok)
            t.check(cell, "stmap_distort_dev frame %d" % frame, got, oracle_stmap_distort(ref, lens, digital, ts, frame))
        if not r["keyed"]:
            frame, ts = r["frames"][0]
            for per_frame in (True, False):
                nw, nh, want_dist, want_und = oracle_stmap(scp, lens, digital, ts, frame, per_frame)
                try:
                    dist, und = dg.generate_stmap(lens, digital, ts, frame, per_frame)
                except g.GyroflowCoreError as e:
                    # the undistort map is the warp's, which has no kernel for (gopro, digital_stretch)
                    if (lens, digital) not in REFERENCE_PAIRS:
                        t.require(cell, "generate_stmap: %s" % e, e.code == GF_ERR_UNSUPPORTED_COMBO)
                    else:
                        t.require(cell, "generate_stmap refused a %dx%d undistorted size: %s" % (nw, nh, e), want_dist is None)
                    continue
                t.require(cell, "generate_stmap of a pair the warp does not compile", (lens, digital) in REFERENCE_PAIRS)
                t.require(cell, "generate_stmap accepted a %dx%d undistorted size" % (nw, nh), want_dist is not None)
                if want_dist is None:
                    continue
                t.check(cell, "generate_stmap per_frame=%d redistort map" % per_frame, dist, want_dist)
                t.check(cell, "generate_stmap per_frame=%d undistort map" % per_frame, und, want_und)
    finally:
        dg.close()
    t.cells.add(cell)


@pytest.mark.gpu
def test_point_path_pairs_and_unsupported_combos():
    """The point path accepts exactly POINT_PAIRS; every other (lens, digital lens) is refused by undistort_points, find_fovs and
    stmap_distort_dev with GF_ERR_UNSUPPORTED_COMBO."""
    import torch
    cp = make_cp(w=64, h=36)
    dg = g.DeviceGyro(cp)
    lib = dg._lib
    pts = np.array([[10.0, 10.0]], np.float32); out = np.zeros_like(pts)
    ts = np.array([100.0]); fov = np.zeros(1)
    buf = torch.zeros(64 * 36 * 3, dtype=torch.float32, device="cuda")
    accepted = []
    names = {v: k for k, v in abi.LENS.items()}
    try:
        for lens in range(len(abi.LENS)):
            for dig in range(len(abi.LENS)):
                rcs = (lib.gf_cuda_undistort_points(dg._h, C.byref(cp.c), lens, dig, 100.0, 0, 0, 1.0, pts.ctypes.data, 1, out.ctypes.data, None),
                       lib.gf_cuda_find_fovs(dg._h, C.byref(cp.c), lens, dig, ts.ctypes.data, 1, 2.0, fov.ctypes.data, None),
                       lib.gf_cuda_stmap_distort_dev(dg._h, C.byref(cp.c), lens, dig, 100.0, 0, buf.data_ptr(), None))
                torch.cuda.synchronize()
                assert rcs in ((0, 0, 0), (GF_ERR_UNSUPPORTED_COMBO,) * 3), (names[lens], names[dig], rcs)
                if rcs == (0, 0, 0):
                    accepted.append((names[lens], names[dig] if dig else None))
    finally:
        dg.close()
    assert sorted(accepted, key=str) == sorted(POINT_PAIRS, key=str) and len(accepted) == 22, accepted


@pytest.mark.gpu
def test_rotation_free_matrix(request):
    """Every pair x every option row with suppress_rotation set: undistort_points, find_fovs, stmap_distort_dev, generate_stmap and
    calculate_fovs bit for bit against the oracle."""
    t0 = time.perf_counter()
    t = Tally()
    want_cells = set()
    for r in ROWS:
        t1 = time.perf_counter()
        for lens, digital in row_pairs(r):
            want_cells.add((lens, digital, r["name"]))
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                run_cell(t, r, lens, digital)
        report(request, "  row %-30s %2d pairs, %.1f s" % (r["name"], len(row_pairs(r)), time.perf_counter() - t1))
    report(request, "test_rotation_free_matrix: %d cells (%d pairs, %d option rows), %d comparisons, %d failing in %d cells, %.1f s" %
           (len(t.cells), len({c[:2] for c in t.cells}), len(ROWS), t.checks, len(t.bad), len(t.bad_cells), time.perf_counter() - t0))
    for c in sorted(t.bad_cells, key=str)[:64]:
        report(request, "  failing cell: %s %s %s" % c)
    for b in t.bad[:64]:
        report(request, "  failing: " + b)
    assert not t.bad, "%d failing comparisons; first: %s" % (len(t.bad), t.bad[0])
    assert t.cells == want_cells and len({c[:2] for c in t.cells}) == 22


@pytest.mark.gpu
def test_large_stmap_and_tiny_frame():
    """stmap_distort_dev on one 3840 x 2160 map and on a 4 x 4 frame (generate_stmap's smallest), bit for bit."""
    from tests.test_stmap import oracle_stmap
    for (w, h), lens, digital in (((3840, 2160), "opencv_fisheye", None), ((4, 4), "sony", "digital_stretch"), ((4, 4), "gopro", "gopro_warp")):
        cp = make_cp(w=w, h=h, lens=lens, digital=digital, camera_stab=_zoom_stab(2, h))
        cp.c.suppress_rotation = 1
        dg = g.DeviceGyro(cp)
        try:
            got, tail_ok = device_stmap_distort(dg, lens, digital, 700.0, 1)
            assert tail_ok, (w, h)
            want = oracle_stmap_distort(cp, lens, digital, 700.0, 1)
            assert same_bits(got, want).all(), ((w, h, lens, digital), first_diff(got, want))
            if w == 4:
                nw, nh, want_dist, want_und = oracle_stmap(cp, lens, digital, 700.0, 1, True)
                dist, und = dg.generate_stmap(lens, digital, 700.0, 1, True)
                assert same_bits(dist, want_dist).all() and same_bits(und, want_und).all(), (lens, digital)
        finally:
            dg.close()


LENS_A = dict(camera_matrix=[900.0, 0.0, 955.0, 0.0, 905.0, 545.0, 0.0, 0.0, 1.0], distortion_coeffs=[0.05, -0.02, 0.004, -0.001] + [0.0] * 8)
LENS_B = dict(camera_matrix=[1100.0, 0.0, 965.0, 0.0, 1090.0, 530.0, 0.0, 0.0, 1.0], distortion_coeffs=[0.02, 0.01, -0.003, 0.0005] + [0.0] * 8)


def _scaled(lens_data, w, h):
    """lens_data for a w x h frame instead of 1920 x 1080."""
    k = list(lens_data["camera_matrix"])
    k[0] *= w / 1920.0; k[2] *= w / 1920.0; k[4] *= h / 1080.0; k[5] *= h / 1080.0
    return dict(lens_data, camera_matrix=k)


def _lens_cp(lens, w, h, lens_data=None, lens_per_frame=None):
    cp = make_cp(w=w, h=h, lens=lens, lens_per_frame=lens_per_frame, params=dict(lens_correction_amount=0.6))
    if lens_data:
        cp.c.camera_matrix[:] = lens_data["camera_matrix"]; cp.c.distortion_coeffs[:] = lens_data["distortion_coeffs"]
    cp.c.suppress_rotation = 1
    return cp


@pytest.mark.gpu
@pytest.mark.parametrize("lens", ["opencv_fisheye", "sony"])
def test_per_frame_lens_data(lens):
    """Per-frame lens data on the point path (resolve_point_lens): undistort_points and stmap_distort_dev for frame i equal the same
    calls on a ComputeParams whose constants are frame i's lens, and that ComputeParams' oracle run, bit for bit."""
    sw, sh = STMAP_SIZE
    per_frame = [LENS_A, LENS_B]
    pts = point_set(1920, 1080, 1031)
    dg = g.DeviceGyro(_lens_cp(lens, 1920, 1080, lens_per_frame=per_frame))
    sdg = g.DeviceGyro(_lens_cp(lens, sw, sh, lens_per_frame=[_scaled(L, sw, sh) for L in per_frame]))
    try:
        outs = []
        for frame, ts in ((0, 400.0), (1, 1800.0)):
            const = _lens_cp(lens, 1920, 1080, per_frame[frame])
            got = dg.undistort_points(lens, None, pts, ts, frame=frame, lens_correction_amount=0.6)
            cdg = g.DeviceGyro(const)
            want_dev = cdg.undistort_points(lens, None, pts, ts, frame=frame, lens_correction_amount=0.6)
            cdg.close()
            want = oracle_points(const, lens, None, pts, ts, frame, 0.6, False)
            assert same_bits(got, want_dev).all(), (frame, first_diff(got, want_dev))
            assert same_bits(got, want).all(), (frame, first_diff(got, want))
            outs.append(got)
            got_map, tail_ok = device_stmap_distort(sdg, lens, None, ts, frame)
            assert tail_ok
            want_map = oracle_stmap_distort(_lens_cp(lens, sw, sh, _scaled(per_frame[frame], sw, sh)), lens, None, ts, frame)
            assert same_bits(got_map, want_map).all(), (frame, first_diff(got_map, want_map))
        assert not same_bits(outs[0], outs[1]).all()
        # DESIGN §8: find_fov does not read the per-frame lens yet; it keeps the constant lens.  This pins today's behaviour, so the
        # change that makes find_fovs follow the per-frame lens has to update this assertion on purpose.
        ts = np.array([400.0, 1800.0])
        pdg = g.DeviceGyro(_lens_cp(lens, 1920, 1080))
        without = pdg.find_fovs(lens, None, ts)
        pdg.close()
        assert same_bits(dg.find_fovs(lens, None, ts), without).all()
    finally:
        dg.close(); sdg.close()


@pytest.mark.gpu
def test_rotation_on_cells(request):
    """Every pair once with the rotation, rolling shutter and IBIS on.  The rotation's f64 acos / sin differ by an ulp between the
    device and glibc, so these keep the bars of the rotation: FOVs to a relative 1e-6, in-frame points to 2e-3 px, and at least 90 % of
    all values bit-identical.  Off-frame points, up to 1e30 away, amplify an ulp of the rotation past any fixed bar: they count towards
    the bit-identical share and must be NaN exactly where the oracle's are."""
    w, h = 1920, 1080
    pts = point_set(w, h)
    inside = (pts[:, 0] >= 0) & (pts[:, 0] <= w) & (pts[:, 1] >= 0) & (pts[:, 1] <= h)
    ts = np.array([-50.0, 300.0, 1234.5, 1234.5, 2100.0, 2900.0, 3500.0, DURATION_MS + 100.0])
    failures = []
    for lens, digital in POINT_PAIRS:
        cp = make_cp(lens=lens, digital=digital, camera_stab=_zoom_stab(8, h), params=dict(lens_correction_amount=0.8))
        dg = g.DeviceGyro(cp)
        same, total, worst_px, worst_rel = 0, 0, 0.0, 0.0
        try:
            for frame in (1, 5):
                got = dg.undistort_points(lens, digital, pts, ts[frame], frame=frame, lens_correction_amount=0.8)
                want = oracle_points(cp, lens, digital, pts, ts[frame], frame, 0.8, False)
                same += int(same_bits(got, want).sum()); total += got.size
                d = np.abs(got[inside] - want[inside])
                worst_px = max(worst_px, float(np.nanmax(d)))
                if not np.allclose(got[inside], want[inside], rtol=0, atol=2e-3, equal_nan=True):
                    failures.append("%s frame %d: in-frame point off by %g px" % ((lens, digital), frame, float(np.nanmax(d))))
                if not (np.isnan(got[~inside]) == np.isnan(want[~inside])).all():
                    failures.append("%s frame %d: an off-frame point is NaN on one side only" % ((lens, digital), frame))
            got = dg.find_fovs(lens, digital, ts)
            want = oracle_lib.find_fovs(cp, lens, digital, ts)
            same += int(same_bits(got, want).sum()); total += got.size
            worst_rel = float(np.abs(got / want - 1).max())
            if not np.allclose(got, want, rtol=1e-6, atol=0):
                failures.append("%s find_fovs off by %g relative" % ((lens, digital), worst_rel))
        finally:
            dg.close()
        share = same / total
        report(request, "  rotation on %-40s %6.2f %% bit-identical, largest in-frame point difference %.3g px, largest FOV difference %.3g" %
               ((lens, digital), 100.0 * share, worst_px, worst_rel))
        if share < 0.9:
            failures.append("%s only %.1f %% bit-identical" % ((lens, digital), 100.0 * share))
    assert not failures, failures


# ---- the second transcription, without a GPU -------------------------------------------------------------------------------------
def cpu_points(w, h):
    """A reduced point set for the pure-Python transcription: the principal point, an axis point, corners, an off-frame point and a
    far one, and -0.0."""
    return np.asarray([(w / 2.0, h / 2.0), (w / 2.0 + 0.3 * w, h / 2.0), (0, 0), (w, h), (w - 1, 3), (-0.2 * w, 1.2 * h), (40.0 * w, 30.0 * h),
                       (-0.0, -0.0)], np.float32)


def test_oracle_matches_second_restatement():
    """The oracle's undistort_points == tests/np_zoom.py bit for bit, for every pair and every option row the transcription covers
    (it has no keyframes), with the rotation suppressed and on; find_fov of one frame per pair and row with the rotation
    suppressed."""
    from tests import np_zoom
    checked, bad = 0, []
    for r in ROWS:
        if not r["np_zoom"]:
            continue
        w, h = min(r["size"][0], 1920), min(r["size"][1], 1920)
        for lens, digital in row_pairs(r):
            for suppress in (True, False):
                cp = build_cp(r, lens, digital, w, h, suppress=suppress)
                kw = r["kw"](w, h)
                stabs, meshes = kw.get("camera_stab"), kw.get("distorting_meshes")
                lca = float(cp.c.lens_correction_amount)
                pts = cpu_points(w, h)
                for frame, ts in r["frames"][:2]:
                    want = oracle_points(cp, lens, digital, pts, ts, frame, lca, r["use_fovs"])
                    stab = stabs[frame] if stabs and frame < len(stabs) else None
                    mesh = meshes[frame] if meshes and frame < len(meshes) else None
                    mesh = None if mesh is None else [float(v) for v in mesh]
                    with warnings.catch_warnings():
                        warnings.simplefilter("ignore")
                        got = np.array(np_zoom.undistort_points_with_rolling_shutter(cp, [tuple(p) for p in pts], ts, frame, lca, r["use_fovs"], lens, digital,
                                                                                      stab, mesh), np.float32)
                    checked += 1
                    if not same_bits(got, want).all():
                        bad.append("%s %s rotation %s frame %d: %s" % ((lens, digital), r["name"], "off" if suppress else "on", frame, first_diff(got, want)))
                if suppress and not stabs and not meshes:
                    frame, ts = 0, r["fov_ts"][1]
                    org = (cp.c.output_width, cp.c.output_height)
                    want = oracle_lib.find_fovs(cp, lens, digital, [ts], r["margins"][-1])[0]
                    adj = build_cp(r, lens, digital, w, h)
                    adj.c.fov_scale = 1.0; adj.c.n_fovs = 0; adj.c.n_minimal_fovs = 0; adj.c.output_width = adj.c.width; adj.c.output_height = adj.c.height
                    with warnings.catch_warnings():
                        warnings.simplefilter("ignore")
                        got = np_zoom.find_fov(adj, org, ts, frame, margin=r["margins"][-1], lens=lens, digital=digital)
                    checked += 1
                    if got != want:
                        bad.append("%s %s find_fov: %r != %r" % ((lens, digital), r["name"], got, want))
    assert not bad, "%d of %d comparisons differ; first: %s" % (len(bad), checked, bad[0])
