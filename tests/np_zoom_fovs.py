"""Second, independent restatement of zooming::calculate_fovs after find_fov — TEST INFRASTRUCTURE ONLY.

  calculate_fovs    <- the trim-range fill of FovIterative::compute   src/core/zooming/fov_iterative.rs:59-69
                       the zoom mode                                   src/core/zooming/mod.rs:55-68
                       zoom_dynamic::compute, both branches            src/core/zooming/zoom_dynamic.rs:15-189

Written from the Rust text in Python floats (= f64).  The keyframe tracks are evaluated with tests/np_producer.keyframe_value_at, and
min_rolling_dynamic / convolve_dynamic / the per-frame-alpha envelope_follower are transcribed literally; the static-window branch is
tests/np_zoom.zoom_dynamic.  The library (gf_zoom_fovs) and the C oracle (oracle/gf_oracle_zoom.c) are checked against it in
tests/test_zoom_fovs.py.
"""
import math

from tests import np_producer
from tests.np_zoom import zoom_dynamic


def _as_usize(x):                                                                  # `f64 as usize`: truncate, saturate, NaN -> 0
    if math.isnan(x) or x <= 0.0:
        return 0
    return min(int(x), (1 << 64) - 1)


def _frames_per_window(window, fps):                                              # get_frames_per_window :82-88 (the GLOBAL window)
    frames = _as_usize(math.floor(window * fps))
    return frames + 1 if frames % 2 == 0 else frames


def _pad_edge(arr, pad):                                                          # :114-125
    return [arr[0]] * pad + list(arr) + [arr[-1]] * pad


def _gaussian_window_normalized(m):                                               # :102-112, std = m / 6
    std = m / 6.0
    sig2 = 2.0 * std * std
    w = [math.exp(-float(x * x) / sig2) for x in range(-(m // 2), m // 2 + 1)]
    s = 0.0
    for t in w: s += t
    return [t / s for t in w]


def _min_rolling_dynamic(a, max_window_half, data):                               # :129-143
    ret = []
    for di, d in enumerate(data):
        i = di + (max_window_half - d["half_frames"])
        if i >= 0 and i + d["frames"] <= len(a):
            ret.append(min(a[i:i + d["frames"]]))
    return ret


def _convolve_dynamic(a, max_window_half, data):                                  # :145-163
    ret = []
    for di, d in enumerate(data):
        i = di + (max_window_half - d["half_frames"])
        if i >= 0 and i + d["frames"] <= len(a):
            acc = 0.0
            for x, y in zip(a[i:i + d["frames"]], d["gaussian_window"]): acc += x * y
            ret.append(acc)
    return ret


def _envelope_follower_dynamic(a, data, alpha):                                   # :165-189 (alpha None: each frame's own)
    alphas = [alpha] * len(a) if alpha is not None else [1.0 - math.exp(-(1.0 / d["fps"]) / d["window"]) for d in data]
    q = a[-1]
    rev = []
    for x, c in reversed(list(zip(a, alphas))):
        q = min(x, x * c + q * (1.0 - c))
        rev.append(q)
    q = rev[-1]
    out = []
    for x, c in zip(reversed(rev), alphas):
        q = min(x, x * c + q * (1.0 - c))
        out.append(q)
    return out


def calculate_fovs(fov_values, timestamps_ms, adaptive_zoom_window, method, scaled_fps, video_speed=1.0, video_speed_affects_zooming=False,
                   zooming_speed=(), video_speed_keys=(), timestamp_scale=None, trim_ranges=()):
    """calculate_fovs from the per-frame find_fov values on: returns (fovs, minimal_fovs).  zooming_speed / video_speed_keys:
    [(timestamp_us, value, easing name)] KeyframeManager tracks, evaluated with np_producer.keyframe_value_at."""
    v = [float(x) for x in fov_values]
    if not v:
        return [], []                                                              # mod.rs:36-38
    l = float(len(v) - 1)
    if trim_ranges and v:                                                          # fov_iterative.rs:59-69
        max_fov = max(v)
        for i in range(len(v)):
            if not any(i >= _as_usize(math.floor(l * r0)) and i <= _as_usize(math.ceil(l * r1)) for r0, r1 in trim_ranges):
                v[i] = max_fov
    if adaptive_zoom_window < -0.9:                                                # mod.rs:55-61: static zoom
        return [min(v)] * len(v), v
    if not adaptive_zoom_window > 0.0001:                                          # :65-67: disabled
        return [1.0] * len(v), v
    minimal = list(v)                                                              # zoom_dynamic.rs:18
    if zooming_speed or (video_speed_affects_zooming and (video_speed != 1.0 or video_speed_keys)):      # :22 keyframed window
        data = []
        max_window = 0
        for ts in timestamps_ms:                                                   # :25-40
            w = np_producer.keyframe_value_at(list(zooming_speed), ts, timestamp_scale)
            w = adaptive_zoom_window if w is None else w
            if video_speed_affects_zooming:
                s = np_producer.keyframe_value_at(list(video_speed_keys), ts, timestamp_scale)
                w *= abs(video_speed if s is None else s)
            frames = _frames_per_window(adaptive_zoom_window, scaled_fps)
            max_window = max(max_window, frames)
            data.append(dict(window=w, fps=scaled_fps, frames=frames, half_frames=frames // 2, gaussian_window=_gaussian_window_normalized(frames)))
        if method == 1:                                                            # :50-54
            second = 1.0 - math.exp(-(1.0 / scaled_fps) / 0.2)
            v = _envelope_follower_dynamic(v, data, None)
            v = _envelope_follower_dynamic(v, data, second)
        else:                                                                      # :43-49
            mwh = max_window // 2
            fov_min = _min_rolling_dynamic(_pad_edge(v, mwh), mwh, data)
            v = _convolve_dynamic(_pad_edge(fov_min, mwh), mwh, data)
        return v, minimal
    return zoom_dynamic(v, adaptive_zoom_window, scaled_fps, 1 if method == 1 else 0), minimal      # :56-76
