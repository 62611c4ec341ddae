"""zooming::calculate_fovs (src/core/zooming/mod.rs:35-70): the trim-range fill (fov_iterative.rs:59-69), the zoom mode (static /
dynamic / disabled) and both branches of zoom_dynamic::compute (zoom_dynamic.rs:15-189), on the host (gf_zoom_fovs) and after the device
find_fov pass (gf_cuda_calculate_fovs).

Three transcriptions agree bit for bit on the host: the library, the C oracle (oracle/gf_oracle_zoom.c: gf_oracle_zoom_fovs, which takes
each frame's ZoomingSpeed / VideoSpeed value as a number; the tracks are evaluated here with tests/np_producer.keyframe_value_at) and
tests/np_zoom_fovs.calculate_fovs (which evaluates the tracks itself and transcribes min_rolling_dynamic / convolve_dynamic literally)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi, synth
from tests import cases, np_producer, np_zoom_fovs, oracle_lib

EASINGS = ("NoEasing", "EaseIn", "EaseOut", "EaseInOut")
FPS = 30.0


_zoom_oracle = None


def _oracle():
    """oracle/libgf_oracle_zoom.so (built by __graft_entry__.build(); rebuilt here when its sources are newer, like oracle_lib.load)."""
    global _zoom_oracle
    if _zoom_oracle is not None:
        return _zoom_oracle
    oracle_lib.load()                                       # libgf_oracle.so, which the zoom module links against, is current
    path = os.path.join(oracle_lib.ORACLE_DIR, "libgf_oracle_zoom.so")
    srcs = ("gf_oracle_zoom.c", "gf_oracle_zoom.h", "gf_oracle.h", "libgf_oracle.so")
    if not os.path.exists(path) or os.path.getmtime(path) < max(os.path.getmtime(os.path.join(oracle_lib.ORACLE_DIR, f)) for f in srcs):
        subprocess.check_call(["make", "-C", oracle_lib.ORACLE_DIR, "-s", "-f", "zoom.mk"])
    lib = C.CDLL(path)
    P = C.POINTER
    lib.gf_oracle_zoom_fovs.restype = None
    lib.gf_oracle_zoom_fovs.argtypes = [P(abi.ZoomParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p]
    lib.gf_oracle_calculate_fovs.restype = None
    lib.gf_oracle_calculate_fovs.argtypes = [P(abi.ComputeParams), P(abi.ZoomParams), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p]
    _zoom_oracle = lib
    return lib


def _timestamps(n, fps=FPS):
    return np.arange(n) * (1000.0 / fps)          # recompute_adaptive_zoom_static (lib.rs:520)


def _fov_values(n, seed=1):
    rng = np.random.default_rng(seed)
    return 0.8 + 0.25 * rng.random(n) + 0.05 * np.sin(np.arange(n) / 7.0)


def _per_frame(kw, ts):
    """The oracle's per-frame inputs: ZoomingSpeed / VideoSpeed at each timestamp, the scalar where a track has no key."""
    scale = kw.get("keyframe_timestamp_scale") or None
    zs, vs = list(kw.get("zooming_speed", ())), list(kw.get("video_speed_keys", ()))
    window, speed = [], []
    for t in ts:
        w = np_producer.keyframe_value_at(zs, float(t), scale) if zs else None
        s = np_producer.keyframe_value_at(vs, float(t), scale) if vs else None
        window.append(kw["adaptive_zoom_window"] if w is None else w)
        speed.append(kw.get("video_speed", 1.0) if s is None else s)
    return np.asarray(window, np.float64), np.asarray(speed, np.float64), int(bool(zs)), int(bool(vs))


def oracle_zoom_fovs(kw, ts, fov):
    fov = np.ascontiguousarray(fov, np.float64)
    window, speed, zk, sk = _per_frame(kw, ts)
    zp = g.ZoomParams(**kw)
    out, minimal = np.zeros_like(fov), np.zeros_like(fov)
    _oracle().gf_oracle_zoom_fovs(C.byref(zp.c), fov.ctypes.data, window.ctypes.data, speed.ctypes.data, zk, sk, fov.size, out.ctypes.data, minimal.ctypes.data)
    return out, minimal


def transcription_fovs(kw, ts, fov):
    out, minimal = np_zoom_fovs.calculate_fovs(fov, [float(t) for t in ts], kw["adaptive_zoom_window"], kw.get("method", 0), kw.get("scaled_fps", 30.0),
                                          video_speed=kw.get("video_speed", 1.0), video_speed_affects_zooming=kw.get("video_speed_affects_zooming", False),
                                          zooming_speed=kw.get("zooming_speed", ()), video_speed_keys=kw.get("video_speed_keys", ()),
                                          timestamp_scale=kw.get("keyframe_timestamp_scale") or None, trim_ranges=kw.get("trim_ranges", ()))
    return np.asarray(out, np.float64), np.asarray(minimal, np.float64)


def _zs_track(easing_a, easing_b=None):
    """A ZoomingSpeed track (seconds) over a 3 s clip whose keys carry the given easings."""
    eb = easing_b or easing_a
    return [(0, 0.4, easing_a), (900_000, 2.5, eb), (1_800_000, 0.8, easing_a), (2_700_000, 1.6, eb)]


SPEED_KEYS = [(0, 1.0, "NoEasing"), (700_000, -2.0, "EaseInOut"), (1_600_000, 0.5, "EaseIn"), (2_500_000, -0.75, "EaseOut")]
CASES = []
for _w in (-1.0, -0.9, 0.0, 0.0001, 2.0):                                      # the mode thresholds of zooming/mod.rs:55-68
    for _m in (0, 1):
        CASES.append(("window%g-m%d" % (_w, _m), 90, dict(adaptive_zoom_window=_w, method=_m, scaled_fps=FPS)))
for _w, _fps in ((0.5, 30.0), (0.4, 30.0), (1.0, 29.97), (0.3, 60.0)):      # 15 (odd), 12 (even), 29 (odd), 18 (even) frames per window
    for _m in (0, 1):
        CASES.append(("frames-%g@%g-m%d" % (_w, _fps, _m), 90, dict(adaptive_zoom_window=_w, method=_m, scaled_fps=_fps)))
for _n in (1, 2):
    for _w in (-1.0, 0.0, 1.0):
        for _m in (0, 1):
            CASES.append(("n%d-window%g-m%d" % (_n, _w, _m), _n, dict(adaptive_zoom_window=_w, method=_m, scaled_fps=FPS)))
    CASES.append(("n%d-trim" % _n, _n, dict(adaptive_zoom_window=1.0, scaled_fps=FPS, trim_ranges=[(1.0, 1.0)])))
    CASES.append(("n%d-keyed" % _n, _n, dict(adaptive_zoom_window=1.0, method=1, scaled_fps=FPS, zooming_speed=_zs_track("EaseIn"))))
TRIMS = {"one": [(0.2, 0.5)], "two": [(0.0, 0.3), (0.6, 0.9)], "overlapping": [(0.1, 0.5), (0.4, 0.7)], "whole": [(0.0, 1.0)],
         "touching-ends": [(0.001, 0.45), (0.55, 0.999)], "beyond-ends": [(-0.5, 0.1), (0.95, 3.0)], "empty-middle": [(0.5, 0.5)]}
for _name, _tr in TRIMS.items():
    for _w, _m in ((-1.0, 0), (0.0, 0), (1.5, 0), (1.5, 1)):
        CASES.append(("trim-%s-window%g-m%d" % (_name, _w, _m), 90, dict(adaptive_zoom_window=_w, method=_m, scaled_fps=FPS, trim_ranges=_tr)))
for _ea in EASINGS:                                                             # ZoomingSpeed keys with every easing
    for _eb in EASINGS:
        CASES.append(("zooming-speed-%s-%s" % (_ea, _eb), 90, dict(adaptive_zoom_window=1.0, method=1, scaled_fps=FPS, zooming_speed=_zs_track(_ea, _eb))))
    CASES.append(("zooming-speed-%s-gaussian" % _ea, 90, dict(adaptive_zoom_window=1.0, method=0, scaled_fps=FPS, zooming_speed=_zs_track(_ea))))
CASES += [
    ("zooming-speed-timestamp-scale", 90, dict(adaptive_zoom_window=1.0, method=1, scaled_fps=FPS, zooming_speed=_zs_track("EaseOut", "EaseIn"), keyframe_timestamp_scale=1.25)),
    ("zooming-speed-one-key", 90, dict(adaptive_zoom_window=1.0, method=1, scaled_fps=FPS, zooming_speed=[(500_000, 0.3, "NoEasing")])),
    ("video-speed-0.5", 90, dict(adaptive_zoom_window=1.0, method=1, scaled_fps=FPS, video_speed=0.5, video_speed_affects_zooming=True)),
    ("video-speed-0.5-gaussian", 90, dict(adaptive_zoom_window=1.0, method=0, scaled_fps=FPS, video_speed=0.5, video_speed_affects_zooming=True)),
    ("video-speed-keys", 90, dict(adaptive_zoom_window=1.0, method=1, scaled_fps=FPS, video_speed_keys=SPEED_KEYS, video_speed_affects_zooming=True)),
    ("video-speed-keys-gaussian", 90, dict(adaptive_zoom_window=1.0, method=0, scaled_fps=FPS, video_speed_keys=SPEED_KEYS, video_speed_affects_zooming=True)),
    ("video-speed-keys-and-zooming-speed", 90, dict(adaptive_zoom_window=1.0, method=1, scaled_fps=FPS, video_speed=0.5, video_speed_keys=SPEED_KEYS[:2],
                                                     video_speed_affects_zooming=True, zooming_speed=_zs_track("EaseInOut"))),
    ("video-speed-keys-not-affecting", 90, dict(adaptive_zoom_window=1.0, method=1, scaled_fps=FPS, video_speed=0.5, video_speed_keys=SPEED_KEYS)),
    ("video-speed-keys-not-affecting-gaussian", 90, dict(adaptive_zoom_window=1.0, method=0, scaled_fps=FPS, video_speed_keys=SPEED_KEYS)),
    ("keyed-trimmed", 90, dict(adaptive_zoom_window=1.0, method=1, scaled_fps=FPS, zooming_speed=_zs_track("EaseIn"), trim_ranges=[(0.2, 0.6)])),
]


@pytest.mark.parametrize("n,kw", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_zoom_fovs_matches_oracle_and_second_transcription(n, kw):
    ts, fov = _timestamps(n, kw["scaled_fps"]), _fov_values(n)
    got, got_min = g.zoom_fovs(g.ZoomParams(**kw), ts, fov)
    want, want_min = oracle_zoom_fovs(kw, ts, fov)
    np_want, np_want_min = transcription_fovs(kw, ts, fov)
    assert np.array_equal(want, np_want) and np.array_equal(want_min, np_want_min)
    assert np.array_equal(got, want) and np.array_equal(got_min, want_min)
    if not kw.get("trim_ranges"):
        assert np.array_equal(got_min, fov)


def test_static_window_branch_taken_when_video_speed_does_not_affect_zooming():
    """VideoSpeed keys and video_speed != 1 without video_speed_affects_zooming and without ZoomingSpeed keys: the static-window branch
    (zoom_dynamic.rs:22, :56-76), i.e. exactly gf_zoom_dynamic_compute; with the flag set the result changes."""
    ts, fov = _timestamps(120), _fov_values(120, seed=4)
    for method in (0, 1):
        kw = dict(adaptive_zoom_window=1.0, method=method, scaled_fps=FPS, video_speed=0.5, video_speed_keys=SPEED_KEYS)
        got, _ = g.zoom_fovs(g.ZoomParams(**kw), ts, fov)
        assert np.array_equal(got, g.zoom_dynamic(fov, 1.0, FPS, method))
    affected, _ = g.zoom_fovs(g.ZoomParams(**dict(kw, video_speed_affects_zooming=True)), ts, fov)
    assert not np.array_equal(affected, got)


def test_keyframed_gaussian_branch_equals_static_window():
    """get_frames_per_window reads the global adaptive_zoom_window, not the frame's window (zoom_dynamic.rs:31), so the keyframed gaussian
    branch gives the static branch's values; only the envelope follower's first pass sees the per-frame window (:171-173)."""
    ts, fov = _timestamps(150), _fov_values(150, seed=2)
    static, _ = g.zoom_fovs(g.ZoomParams(adaptive_zoom_window=1.0, method=0, scaled_fps=FPS), ts, fov)
    for keyed in (dict(zooming_speed=_zs_track("EaseInOut")), dict(video_speed=0.5, video_speed_affects_zooming=True),
                  dict(video_speed_keys=SPEED_KEYS, video_speed_affects_zooming=True)):
        got, _ = g.zoom_fovs(g.ZoomParams(adaptive_zoom_window=1.0, method=0, scaled_fps=FPS, **keyed), ts, fov)
        assert np.array_equal(got, static)
        assert np.array_equal(got, transcription_fovs(dict(adaptive_zoom_window=1.0, method=0, scaled_fps=FPS, **keyed), ts, fov)[0])
        env_static, _ = g.zoom_fovs(g.ZoomParams(adaptive_zoom_window=1.0, method=1, scaled_fps=FPS), ts, fov)
        env_keyed, _ = g.zoom_fovs(g.ZoomParams(adaptive_zoom_window=1.0, method=1, scaled_fps=FPS, **keyed), ts, fov)
        assert not np.array_equal(env_keyed, env_static)


def test_second_envelope_pass_uses_fixed_alpha():
    """The keyframed branch's second envelope pass always uses alpha = 1 - exp(-(1/fps)/0.2) (zoom_dynamic.rs:51), not the frame's window:
    a ZoomingSpeed track with one key w gives the static envelope follower with window w, whose second pass uses 0.2 s too (:71)."""
    ts, fov = _timestamps(120), _fov_values(120, seed=3)
    w = 0.7
    got, _ = g.zoom_fovs(g.ZoomParams(adaptive_zoom_window=2.0, method=1, scaled_fps=FPS, zooming_speed=[(0, w, "NoEasing")]), ts, fov)
    assert np.array_equal(got, g.zoom_dynamic(fov, w, FPS, 1))
    data = [dict(fps=FPS, window=w)] * len(fov)
    per_frame_second_pass = np_zoom_fovs._envelope_follower_dynamic(np_zoom_fovs._envelope_follower_dynamic(list(fov), data, None), data, None)
    assert not np.array_equal(got, np.asarray(per_frame_second_pass))


def test_trim_fill_comes_before_the_mode_branch():
    """Trim ranges are applied in FovIterative::compute (fov_iterative.rs:59-69), before calculate_fovs branches on the mode
    (zooming/mod.rs:55-68): the minimal FOVs of a trimmed clip already carry the max-FOV fill, and static zoom takes the minimum of the
    filled values."""
    n = 91
    ts, fov = _timestamps(n), _fov_values(n, seed=5)
    trim = [(0.25, 0.5)]                                               # l = 90: frames 22..45 stay
    inside = np.zeros(n, bool); inside[22:46] = True
    filled = np.where(inside, fov, fov.max())
    for window, method in ((-1.0, 0), (0.0, 0), (1.0, 0), (1.0, 1)):
        got, got_min = g.zoom_fovs(g.ZoomParams(adaptive_zoom_window=window, method=method, scaled_fps=FPS, trim_ranges=trim), ts, fov)
        assert np.array_equal(got_min, filled), window
        if window < -0.9:
            assert np.all(got == fov[inside].min())
        elif window == 0.0:
            assert np.all(got == 1.0)
        else:
            assert np.array_equal(got, g.zoom_dynamic(filled, window, FPS, method))


def test_zoom_fovs_empty_clip_and_bad_arguments():
    lib = abi.load_library()
    zp = g.ZoomParams(adaptive_zoom_window=1.0, scaled_fps=FPS)
    out, mn = np.full(1, -7.0), np.full(1, -7.0)
    assert lib.gf_zoom_fovs(C.byref(zp.c), None, None, 0, out.ctypes.data, mn.ctypes.data) == 0       # calculate_fovs returns empty vectors
    assert out[0] == -7.0 and mn[0] == -7.0
    ts, fov = _timestamps(4), _fov_values(4)
    assert lib.gf_zoom_fovs(None, ts.ctypes.data, fov.ctypes.data, 4, out.ctypes.data, mn.ctypes.data) == -1
    bad = g.ZoomParams(adaptive_zoom_window=1.0, scaled_fps=FPS); bad.c.n_trim_ranges = 1             # ranges announced, none given
    out4, mn4 = np.full(4, -7.0), np.full(4, -7.0)
    assert lib.gf_zoom_fovs(C.byref(bad.c), ts.ctypes.data, fov.ctypes.data, 4, out4.ctypes.data, mn4.ctypes.data) == -1
    huge = g.ZoomParams(adaptive_zoom_window=1e300, scaled_fps=FPS)               # a gaussian window no memory holds: rejected, nothing written
    assert lib.gf_zoom_fovs(C.byref(huge.c), ts.ctypes.data, fov.ctypes.data, 4, out4.ctypes.data, mn4.ctypes.data) == -1
    assert np.all(out4 == -7.0) and np.all(mn4 == -7.0)
    assert lib.gf_cuda_calculate_fovs(None, None, C.byref(zp.c), 1, 0, ts.ctypes.data, 4, out4.ctypes.data, mn4.ctypes.data, None) == -1


def test_zoom_params_struct_size_matches_the_library():
    lib = abi.load_library()
    assert lib.gf_abi_struct_size(9) == C.sizeof(abi.ZoomParams)
    assert lib.gf_abi_struct_size(10) == 0


# ---------------------------------------------------------------------------------------------------- device: find_fov + calculate_fovs

def _make_cp(w=1920, h=1080, lens="opencv_fisheye", digital=None, **kw):
    p = synth.base_kernel_params(w, h, lens=lens, digital_lens=digital)
    org, sm = cases.gyro()
    return g.ComputeParams(p, org, sm, **kw)


MODES = {
    "static": dict(adaptive_zoom_window=-1.0),
    "disabled": dict(adaptive_zoom_window=0.0),
    "dynamic-gaussian": dict(adaptive_zoom_window=1.0, method=0),
    "dynamic-envelope-zooming-speed": dict(adaptive_zoom_window=1.0, method=1, zooming_speed=_zs_track("EaseInOut", "EaseIn")),
    "trimmed": dict(adaptive_zoom_window=0.5, method=0, trim_ranges=[(0.1, 0.4), (0.6, 0.8)]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("lens,digital", [("opencv_fisheye", None), ("opencv_fisheye", "gopro_superview"), ("opencv_standard", "digital_stretch")])
def test_device_calculate_fovs_matches_oracle(lens, digital, mode):
    kw = dict(MODES[mode], scaled_fps=FPS, fov_algorithm_margin=2.0)
    cp = _make_cp(lens=lens, digital=digital)
    n = 90
    ts = _timestamps(n)
    dg = g.DeviceGyro(cp)
    got, got_min = dg.calculate_fovs(lens, digital, g.ZoomParams(**kw), ts)
    dg.close()
    window, speed, zk, sk = _per_frame(kw, ts)
    want, want_min = np.zeros(n), np.zeros(n)
    zp = g.ZoomParams(**kw)
    _oracle().gf_oracle_calculate_fovs(C.byref(cp.c), C.byref(zp.c), abi.LENS[lens], abi.LENS[digital] if digital else 0, ts.ctypes.data,
                                       window.ctypes.data, speed.ctypes.data, zk, sk, n, want.ctypes.data, want_min.ctypes.data)
    # find_fov values agree to the relative 1e-6 of test_device_find_fovs_matches_oracle; the filters keep that bar
    assert np.allclose(got_min, want_min, rtol=1e-6, atol=0), float(np.abs(got_min / want_min - 1).max())
    assert np.allclose(got, want, rtol=1e-6, atol=0), float(np.abs(got / want - 1).max())
    assert np.ptp(want_min) > 1e-3
    if mode == "disabled":
        assert np.all(got == 1.0)


@pytest.mark.gpu
def test_queue_renders_with_calculated_fovs():
    """The INTEGRATION.md flow: gf_cuda_calculate_fovs over the clip, its results into cp.fovs / cp.minimal_fovs, then the render queue.
    Every frame (and its checksum) equals the oracle's render of the table produced for the same FOVs."""
    import torch
    from gyroflow_b200 import render_queue
    from tests.test_render_queue import W, H, _job, _expected
    pix, lens = "RGBA8", "opencv_fisheye"
    n = 6
    fps = 60.0
    ts_of = lambda f: f * (1000.0 / fps)
    zp = g.ZoomParams(adaptive_zoom_window=0.5, method=1, scaled_fps=fps, zooming_speed=[(0, 0.2, "EaseIn"), (80_000, 1.0, "EaseOut")])
    _, cp0, _ = _job()
    dg0 = g.DeviceGyro(cp0)
    fovs, minimal = dg0.calculate_fovs(lens, None, zp, [ts_of(f) for f in range(n)])
    dg0.close()
    assert np.abs(fovs - 1.0).max() > 1e-3                             # the zoom changes the frames
    p, cp, st = _job(fovs=fovs, minimal_fovs=minimal)
    st.adaptive_zoom_window = 0.5
    src = synth.synthetic_frame(W, H, pix, stride=p.stride)
    tsrc = torch.from_numpy(src).cuda()
    outs = [torch.zeros((H, p.output_stride), dtype=torch.uint8, device="cuda") for _ in range(n)]
    bufs = [g.Buffers(g.BufferDescription((W, H, p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                      g.BufferDescription((W, H, p.output_stride), o.data_ptr(), length=o.numel())) for o in outs]
    q = g.RenderQueue(cp, st, lens, None, bufs[0].input, bufs[0].output, depth=3, checksum=True)
    sums = q.render(range(n), ts_of, lambda f: bufs[f])
    q.close()
    dg = g.DeviceGyro(cp)
    mats = torch.zeros((max(W, H), 14), dtype=torch.float32, device="cuda")
    for f in range(n):
        kp_h, _, fov, minimal_fov = cp.at_timestamp(ts_of(f), f)
        assert kp_h.fov == np.float32(fovs[f]) and fov == fovs[f] and minimal_fov == minimal[f]
        want = _expected(p, cp, st, dg, mats, ts_of(f), f, src, pix, lens, None, bufs[f])
        assert np.array_equal(outs[f].cpu().numpy(), want), "frame %d" % f
        assert sums[f] == render_queue.checksum_host(want)
    dg.close()
