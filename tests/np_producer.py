"""numpy (f64) restatement of the reference's per-frame producer — TEST INFRASTRUCTURE (moved out of the product package).

  quat_at_timestamp      <- GyroSource::quat_at_timestamp   src/core/gyro_source/mod.rs:857-879 (+ offset_at_timestamp :884-909)
  frame_matrices         <- FrameTransform::at_timestamp    src/core/stabilization/frame_transform.rs:221-308
  catmull_rom            <- CatmullRom::interpolate         src/core/gyro_source/splines.rs:22-83

It is the second, independent transcription the C++ / CUDA producer (gyroflow_b200/csrc/frame_transform.cu) is checked
against (tests/test_frame_transform.py, <= 1 f32 ulp: numpy's pinv / slerp need not match nalgebra's to the last bit — parity
at that boundary is unpinned, SURVEY §8c), and the source of the synthetic matrix tables of the parity tests (tests/cases.py).
"""
import math

import numpy as np

from gyroflow_b200.synth import q_mul, q_inv


def q_slerp(a, b, t):
    """UnitQuaternion::slerp (nalgebra 0.34): shortest arc, linear fallback never needed for distinct neighbours."""
    d = np.sum(a * b, axis=-1, keepdims=True)
    b = np.where(d < 0.0, -b, b)
    d = np.abs(d)
    d = np.clip(d, -1.0, 1.0)
    hang = np.arccos(d)
    s = np.sqrt(1.0 - d * d)
    t = np.asarray(t)[..., None]
    small = s < 1e-12
    s_safe = np.where(small, 1.0, s)
    ta = np.where(small, 1.0 - t, np.sin((1.0 - t) * hang) / s_safe)
    tb = np.where(small, t, np.sin(t * hang) / s_safe)
    return a * ta + b * tb


def q_to_matrix(q):
    w, i, j, k = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    ww, ii, jj, kk = w * w, i * i, j * j, k * k
    ij, wk, wj, ik, jk, wi = i * j * 2.0, w * k * 2.0, w * j * 2.0, i * k * 2.0, j * k * 2.0, w * i * 2.0
    m = np.empty(q.shape[:-1] + (3, 3))
    m[..., 0, 0] = ww + ii - jj - kk; m[..., 0, 1] = ij - wk;           m[..., 0, 2] = wj + ik
    m[..., 1, 0] = wk + ij;           m[..., 1, 1] = ww - ii + jj - kk; m[..., 1, 2] = jk - wi
    m[..., 2, 0] = ik - wj;           m[..., 2, 1] = wi + jk;           m[..., 2, 2] = ww - ii - jj + kk
    return m



def offset_at_timestamp(offsets, timestamp_ms, scalar_ms=0.0):
    """GyroSource::offset_at_timestamp — gyro_source/mod.rs:884-909.  offsets: {timestamp_us: offset_ms}; with no points the
    scalar offset (gyro_offset_ms) applies."""
    if not offsets:
        return scalar_ms
    ks = sorted(offsets)
    if len(ks) == 1:
        return offsets[ks[0]]
    first_ts, last_ts = ks[0], ks[-1]
    timestamp_us = int(timestamp_ms * 1000.0)            # `as i64`: truncation toward zero
    lookup = max(min(timestamp_us, last_ts - 1), first_ts + 1)
    below = [k for k in ks if k <= lookup]
    k1 = below[-1]
    if k1 == lookup:
        return offsets[k1]
    above = [k for k in ks if k >= lookup]
    if not above:
        return 0.0
    k2 = above[0]
    fract = float(timestamp_us - k1) / float(k2 - k1)
    return offsets[k1] + (offsets[k2] - offsets[k1]) * fract


def quat_at_timestamp(track, timestamp_ms, offsets=None, scalar_offset_ms=0.0):
    """gyro_source/mod.rs:857-879; vectorised over timestamp_ms.  offsets: {timestamp_us: offset_ms} or None (then the scalar
    scalar_offset_ms applies)."""
    self = track
    t = np.atleast_1d(np.asarray(timestamp_ms, dtype=np.float64))
    if offsets or scalar_offset_ms != 0.0:
        t = t - np.array([offset_at_timestamp(offsets, float(v), scalar_offset_ms) for v in t])
    us = t * 1000.0
    lookup = np.clip((np.sign(us) * np.floor(np.abs(us) + 0.5)).astype(np.int64), self.ts[0], self.ts[-1])   # f64::round: half away from zero
    i1 = np.searchsorted(self.ts, lookup, side="right") - 1          # last key <= lookup
    i2 = np.minimum(np.searchsorted(self.ts, lookup, side="left"), len(self.ts) - 1)   # first key >= lookup
    t1, t2 = self.ts[i1], self.ts[i2]
    exact = t1 == lookup
    dt = np.where(exact, 1, t2 - t1).astype(np.float64)
    fract = np.where(exact, 0.0, (lookup - t1).astype(np.float64) / dt)
    out = q_slerp(self.q[i1], self.q[i2], fract)
    out = np.where(exact[:, None], self.q[i1], out)
    return out




def catmull_rom(pos, val, t):
    """CatmullRom::interpolate — gyro_source/splines.rs:22-83.  pos[n] ascending, val[n, 3]; None outside [first, last)."""
    n = len(pos)
    if n < 2 or t != t:
        return None
    i = int(np.searchsorted(pos, t, side="left"))
    if i < n and pos[i] == t:
        if i == n - 1: return None
        lower = i
    else:
        if i >= n or i == 0: return None
        lower = i - 1
    a, b = val[lower], val[lower + 1]
    k = (t - pos[lower]) / (pos[lower + 1] - pos[lower])
    x = a * 2.0 - b if lower == 0 else val[lower - 1]
    y = b * 2.0 - a if lower + 2 >= n else val[lower + 2]
    return ((((a * 3.0 - x) - b * 3.0) + y) * 0.5) * k * k * k + ((b - x) * 0.5) * k + a + (((b * 4.0 + a * -5.0 + x + x) - y) * 0.5) * k * k


def stab_row(stab, y, width, height, framebuffer_inverted):
    """frame_transform.rs:227-236, :269-285 for one row: (sx, sy, ra_rad, ox, oy) in f64."""
    cx, cy, cw, ch = [float(np.float32(v)) for v in stab["crop_area"]]
    pp = stab["pixel_pitch"]
    sc = (width / cw / float(pp[0]), height / ch / float(pp[1]) * (-1.0 if framebuffer_inverted else 1.0))
    y_sensor = (float(y) - 0.0) * ((cy + ch) - cy) / (float(height) - 0.0) + cy
    if framebuffer_inverted:
        y_sensor = float(stab["sensor_size"][1]) - y_sensor
    z = np.zeros(3)
    none = (np.zeros(0), np.zeros((0, 3)))                                 # an entry without a spline has no points
    ibis, ois = stab.get("ibis", none), stab.get("ois", none)
    s = catmull_rom(np.asarray(ibis[0], float), np.asarray(ibis[1], float).reshape(-1, 3), y_sensor + stab.get("offset", 0.0))
    o = catmull_rom(np.asarray(ois[0], float), np.asarray(ois[1], float).reshape(-1, 3), y_sensor + stab.get("offset", 0.0))
    s = z if s is None else s; o = z if o is None else o
    ra = s[2] / 1000.0 * (-1.0 if framebuffer_inverted else 1.0)
    return (s[0] * sc[0], s[1] * sc[1], ra * (math.pi / 180.0), o[0] * sc[0], o[1] * sc[1])


def frame_matrices(p, org, smoothed, timestamp_ms, frame_readout_time_ms=16.0, video_rotation_deg=0.0,
                   horizontal=False, framebuffer_inverted=False, ibis=None, offsets=None, stab=None, fov_f64=None,
                   gyro_offset_ms=0.0, suppress_rotation=False, camera_stab=None, frame=0, camera_matrix=None):
    """FrameTransform::at_timestamp rows — frame_transform.rs:221-308 (f64 -> f32).

    frame_readout_time_ms: the signed, scaled get_frame_readout_time (:22-36).
    ibis: optional callable row -> (sx, sy, ra_rad, ox, oy) filling m[9..13] (synthetic stand-in for the IBIS/OIS splines).
    offsets: multi-point sync offsets {timestamp_us: offset_ms}; without points gyro_offset_ms applies.
    camera_stab: the per-frame CameraStabData list; frame `frame` is used, a frame past its end has none (:227).
    camera_matrix: the frame's K (9 values, row-major) when it is not the KernelParams' f / c."""
    if camera_matrix is None:
        camera_matrix = [float(p.f[0]), 0.0, float(p.c[0]), 0.0, float(p.f[1]), float(p.c[1]), 0.0, 0.0, 1.0]
    K = [float(v) for v in camera_matrix]
    fov = float(p.fov) if fov_f64 is None else float(fov_f64)      # the reference keeps fov in f64 until KernelParams (:191, :329)
    new_k = np.array([[K[0] / fov, K[1], p.output_width / 2.0], [K[3], K[4] / fov, p.output_height / 2.0], [K[6], K[7], K[8]]])   # get_new_k :37-51
    if camera_stab is not None:
        stab = camera_stab[frame] if frame < len(camera_stab) else None
    frt = frame_readout_time_ms
    n = (p.width if horizontal else p.height)
    rows = n if abs(frt) > 0.0 else 1
    row_readout_time = frt / n
    start_ts = timestamp_ms - frt / 2.0
    a = math.radians(video_rotation_deg)
    image_rotation = np.array([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]])
    quat1 = q_inv(quat_at_timestamp(org, timestamp_ms, offsets, gyro_offset_ms)[0])
    sq1 = quat_at_timestamp(smoothed, timestamp_ms, offsets, gyro_offset_ms)[0]
    qt = start_ts + row_readout_time * np.arange(rows) if abs(frt) > 0.0 else np.array([start_ts])
    quat = q_mul(q_mul(sq1[None, :], quat1[None, :]), quat_at_timestamp(org, qt, offsets, gyro_offset_ms))
    r = image_rotation[None] @ q_to_matrix(quat)
    if framebuffer_inverted:
        r[:, 0, 2] *= -1; r[:, 1, 2] *= -1; r[:, 2, 0] *= -1; r[:, 2, 1] *= -1
    else:
        r[:, 0, 1] *= -1; r[:, 0, 2] *= -1; r[:, 1, 0] *= -1; r[:, 2, 0] *= -1
    if suppress_rotation:                                             # :289-290
        r[:] = np.eye(3)
    i_r = np.linalg.pinv(new_k[None] @ r, rcond=1e-6)
    m = np.zeros((rows, 14), dtype=np.float32)
    m[:, :9] = i_r.reshape(rows, 9).astype(np.float32)
    if ibis is not None:
        for y in range(rows):
            m[y, 9:14] = np.asarray(ibis(y), dtype=np.float32)
    if stab is not None:
        for y in range(rows):
            m[y, 9:14] = np.asarray(stab_row(stab, y, p.width, p.height, framebuffer_inverted), dtype=np.float32)
    if suppress_rotation and frt == 0.0:                              # :289-293: no rotation and no rolling shutter, no shifts either
        m[:, 9:14] = 0.0
    return m


def identity_matrices(p, rows=1):
    """Identity quaternions: i_r = inverse(new_k) for every row."""
    fov = float(p.fov)
    new_k = np.array([[p.f[0] / fov, 0.0, p.output_width / 2.0], [0.0, p.f[1] / fov, p.output_height / 2.0], [0.0, 0.0, 1.0]], dtype=np.float64)
    r = np.eye(3); r[0, 1] *= -1; r[0, 2] *= -1; r[1, 0] *= -1; r[2, 0] *= -1
    i_r = np.linalg.pinv(new_k @ r)
    m = np.zeros((rows, 14), dtype=np.float32)
    m[:, :9] = i_r.reshape(1, 9).astype(np.float32)
    return m




# ---- KeyframeManager::value_at_video_timestamp for one track: keyframes.rs:169-205, Easing::get / interpolate :279-303 ----
def _easing_get(a, b):                       # keyframes.rs:279-291 (names as in the enum :74-81)
    a_out = a in ("EaseOut", "EaseInOut")
    b_in = b in ("EaseIn", "EaseInOut")
    if a_out and b_in: return "EaseInOut"
    if b_in: return "EaseOut"
    if a_out: return "EaseIn"
    return "NoEasing"


def _easing_interpolate(e, a, b, x):         # keyframes.rs:292-302; simple_easing 1.0.2 (easings.net sine family) on f32
    import ctypes, ctypes.util
    libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
    libm.cosf.restype = ctypes.c_float; libm.cosf.argtypes = [ctypes.c_float]
    libm.sinf.restype = ctypes.c_float; libm.sinf.argtypes = [ctypes.c_float]
    f = np.float32
    xf = f(x); pi = f(math.pi)
    if e == "EaseIn":      x = float(f(1.0) - f(libm.cosf(float(xf * pi / f(2.0)))))
    elif e == "EaseOut":   x = float(f(libm.sinf(float(xf * pi / f(2.0)))))
    elif e == "EaseInOut": x = float(-(f(libm.cosf(float(pi * xf))) - f(1.0)) / f(2.0))
    return a * (1.0 - x) + b * x


def keyframe_value_at(keys, timestamp_ms, timestamp_scale=None):
    """keys: [(timestamp_us, value, easing name)] in any order (a BTreeMap in the reference).  Returns the value or None."""
    keys = sorted(keys)
    if len(keys) == 0: return None
    if len(keys) == 1: return keys[0][1]
    first_ts, last_ts = keys[0][0], keys[-1][0]
    t = timestamp_ms * 1000.0 * (timestamp_scale if timestamp_scale is not None else 1.0)
    timestamp_us = int(math.copysign(math.floor(abs(t) + 0.5), t))            # f64::round (half away from zero) as i64
    lookup_ts = max(min(timestamp_us, last_ts), first_ts)
    below = [k for k in keys if k[0] <= lookup_ts]
    if not below: return None
    o1 = below[-1]
    if o1[0] == lookup_ts: return o1[1]
    above = [k for k in keys if k[0] >= lookup_ts]
    if not above: return None
    o2 = above[0]
    time_delta = float(o2[0] - o1[0])
    alpha = float(timestamp_us - o1[0]) / time_delta
    return _easing_interpolate(_easing_get(o1[2], o2[2]), o1[1], o2[1], alpha)
