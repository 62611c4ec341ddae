"""Synthetic inputs for tests and bench.py (SURVEY.md §8d): high-entropy frames, a 240 Hz gyro track, lens coefficients, a
9x9 mesh, and a KernelParams template with the reference's defaults.  DATA GENERATORS ONLY: the numpy restatement of the
per-frame producer (FrameTransform::at_timestamp) that round 1 kept here is test infrastructure and lives in
tests/np_producer.py; the product's producer is csrc/frame_transform.cu behind the C ABI.

Quaternions are (w, x, y, z), Hamilton product, like nalgebra's UnitQuaternion<f64>.
"""
import math

import numpy as np

from . import abi

# ------------------------------------------------------------------------------------------ frames


def _hash32(a):
    a = a.astype(np.uint64)
    a = (a ^ (a >> 16)) * np.uint64(0x7feb352d) & np.uint64(0xffffffff)
    a = (a ^ (a >> 15)) * np.uint64(0x846ca68b) & np.uint64(0xffffffff)
    a = a ^ (a >> 16)
    return a.astype(np.uint32)


def synthetic_frame(width, height, pixel_type="RGBA8", frame=0, stride=None, seed=0x9E3779B9):
    """High-entropy frame: value = hash32(seed, frame, byte index) reduced to the format's range.
    Returns a (height, stride) uint8 array (stride defaults to width*bpp rounded up to 256 B)."""
    _, count, sdt = abi.PIXEL_TYPES[pixel_type]
    dt = np.dtype(sdt)
    bpp = count * dt.itemsize
    if stride is None:
        stride = (width * bpp + 255) // 256 * 256
    n_el = height * width * count
    idx = np.arange(n_el, dtype=np.uint64) + np.uint64((seed ^ (frame * 0x85ebca6b)) & 0xffffffff) * np.uint64(0x9E3779B1)
    h = _hash32(idx)
    if dt.kind == "u":
        vals = (h & np.uint32((1 << (8 * dt.itemsize)) - 1)).astype(dt)
    elif dt == np.dtype("f4"):
        vals = ((h >> 8).astype(np.float32) / np.float32(1 << 24)).astype(np.float32)
    else:
        vals = ((h >> 8).astype(np.float32) / np.float32(1 << 24)).astype(np.float16)
    buf = np.zeros((height, stride), dtype=np.uint8)
    buf[:, : width * bpp] = vals.reshape(height, width * count).view(np.uint8).reshape(height, width * bpp)
    return buf


# bit patterns of the special values edge_frame mixes in: NaNs with assorted signs and payloads (quiet and signalling), +-Inf
_NAN_F32 = [0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FA5A5A5, 0xFFFFFFFF, 0x7FFFFFFF]
_NAN_F16 = [0x7E00, 0xFE00, 0x7C01, 0x7D55, 0xFFFF, 0x7FFF]


def edge_frame(width, height, pixel_type, seed=0, stride=None):
    """A frame at the edges of the format's value domain, as a (height, stride) uint8 array like synthetic_frame.

    f32 / f16: ordinary values in [0, 1) mixed with HDR values (1 .. 1e4), values near f16's largest finite 65504 (f16 only),
    negatives, subnormals, +-0, +-Inf and NaNs with assorted payloads.  The non-finite values sit in every fourth 8 x 8 tile only,
    so that most footprints of the 16- and 64-tap resamplers still see finite content.
    u8 / u16: 0 / max checkerboards (pixel parity, flipped per 8 x 8 tile and per channel), which make the bicubic and Lanczos
    taps overshoot hardest."""
    _, count, sdt = abi.PIXEL_TYPES[pixel_type]
    dt = np.dtype(sdt)
    bpp = count * dt.itemsize
    if stride is None:
        stride = (width * bpp + 255) // 256 * 256
    rng = np.random.Generator(np.random.PCG64(seed))
    y, x, c = np.meshgrid(np.arange(height), np.arange(width), np.arange(count), indexing="ij")
    tile = rng.integers(0, 2, size=(height // 8 + 1, width // 8 + 1))[y // 8, x // 8]
    if dt.kind == "u":
        vals = np.where(((x + y + c + tile) & 1) == 1, np.iinfo(dt).max, 0).astype(dt)
    else:
        f16 = dt == np.dtype("f2")
        shape = x.shape
        v = rng.random(shape, dtype=np.float32)                                                  # ordinary
        kind = rng.integers(0, 100, size=shape)
        hdr = np.float32(10.0) ** rng.uniform(0.0, 4.0, shape).astype(np.float32)              # 1 .. 1e4
        v = np.where(kind < 12, hdr, v)
        v = np.where((kind >= 12) & (kind < 24), -v * np.float32(10.0) ** rng.integers(-2, 3, shape).astype(np.float32), v)   # negatives
        tiny = (np.float32(2.0) ** -20 if f16 else np.float32(1e-40)) * rng.integers(1, 16, shape).astype(np.float32)          # subnormals
        v = np.where((kind >= 24) & (kind < 30), np.where(rng.integers(0, 2, shape) == 1, -tiny, tiny), v)
        v = np.where((kind >= 30) & (kind < 34), np.float32(0.0), v)
        v = np.where((kind >= 34) & (kind < 38), np.float32(-0.0), v)
        if f16:
            near = rng.choice(np.array([65504.0, 65472.0, 65440.0, 60000.0, -65504.0], np.float32), size=shape)
            v = np.where((kind >= 38) & (kind < 45), near, v)
        vals = v.astype(dt)
        bits = vals.view(np.uint16 if f16 else np.uint32)
        nonfinite = ((y // 8 + x // 8) % 4 == 0) & (kind >= 88)
        pos_inf, neg_inf = (0x7C00, 0xFC00) if f16 else (0x7F800000, 0xFF800000)
        nans = np.array(_NAN_F16 if f16 else _NAN_F32, dtype=bits.dtype)
        special = np.where(kind >= 96, nans[rng.integers(0, len(nans), shape)], np.where(kind >= 92, neg_inf, pos_inf)).astype(bits.dtype)
        vals = np.where(nonfinite, special, bits).view(dt)
    buf = np.zeros((height, stride), dtype=np.uint8)
    buf[:, : width * bpp] = np.ascontiguousarray(vals).reshape(height, width * count).view(np.uint8).reshape(height, width * bpp)
    return buf


# ------------------------------------------------------------------------------------------ quaternions


def q_mul(a, b):
    aw, ax, ay, az = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bw, bx, by, bz = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([aw * bw - ax * bx - ay * by - az * bz,
                     aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw], axis=-1)


def q_inv(q):
    return q * np.array([1.0, -1.0, -1.0, -1.0])


def q_normalize(q):
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


class GyroTrack:
    """`TimeQuat = BTreeMap<i64 us, UnitQuaternion<f64>>` as sorted arrays (gyro_source/mod.rs:34)."""

    def __init__(self, ts_us, quats):
        self.ts = np.asarray(ts_us, dtype=np.int64)
        self.q = np.asarray(quats, dtype=np.float64)


def synthetic_gyro(duration_s, rate_hz=240.0, seed=42):
    """org track = integrated omega(t) = (0.30 sin 2pi 1.3t, 0.22 sin 2pi 0.7t + 0.05, 0.15 sin 2pi 2.1t) rad/s + N(0, 0.02);
    smoothed track = the reference's stored form smooth^-1 * org (gyro_source/mod.rs:682-685), smooth = 1 s box filter."""
    n = int(duration_s * rate_hz) + 1
    dt = 1.0 / rate_hz
    t = np.arange(n) * dt
    rng = np.random.Generator(np.random.PCG64(seed))
    w = np.stack([0.30 * np.sin(2 * np.pi * 1.3 * t), 0.22 * np.sin(2 * np.pi * 0.7 * t) + 0.05, 0.15 * np.sin(2 * np.pi * 2.1 * t)], axis=1)
    w = w + rng.normal(0.0, 0.02, size=w.shape)
    q = np.empty((n, 4)); q[0] = [1.0, 0.0, 0.0, 0.0]
    ang = np.linalg.norm(w, axis=1) * dt
    axis = w / np.maximum(np.linalg.norm(w, axis=1, keepdims=True), 1e-30)
    dq = np.concatenate([np.cos(ang / 2)[:, None], axis * np.sin(ang / 2)[:, None]], axis=1)
    for i in range(1, n):
        q[i] = q_mul(q[i - 1], dq[i - 1])
    q = q_normalize(q)
    # hemisphere-continuous copy for the box filter
    qc = q.copy()
    for i in range(1, n):
        if np.dot(qc[i], qc[i - 1]) < 0:
            qc[i] = -qc[i]
    half = int(rate_hz // 2)
    csum = np.concatenate([np.zeros((1, 4)), np.cumsum(qc, axis=0)], axis=0)
    lo = np.maximum(np.arange(n) - half, 0); hi = np.minimum(np.arange(n) + half + 1, n)
    smooth = q_normalize(csum[hi] - csum[lo])
    stored = q_normalize(q_mul(q_inv(smooth), q))
    ts_us = np.round(t * 1e6).astype(np.int64)
    return GyroTrack(ts_us, q), GyroTrack(ts_us, stored)


# ------------------------------------------------------------------------------------------ lens / params

# synthetic coefficients (no lens profiles are vendored in the reference, core/build.rs:4-17)
LENS_COEFFS = {
    "opencv_fisheye": [0.04, -0.01, 0.002, -0.0005],
    "opencv_standard": [-0.12, 0.05, 0.0008, -0.0006, -0.01, 0.02, 0.01, 0.002, 0.0003, -0.0002, 0.0002, -0.0001],
    "poly3": [0.02],
    "poly5": [0.015, 0.004],
    "ptlens": [0.006, -0.01, 0.02],
    "insta360": [0.03, -0.008, 0.002, 0.0005, -0.0004, 0.9],
    "sony": [1.0, 0.02, -0.03, 0.01, 0.0, 0.0],
    "generic_polynomial": [1.0, 0.01, -0.04, 0.01, 0.004, -0.002, 0.001, 0.0, 0.0, 0.0, 0.0, 0.0],
    "gopro": [0.0, 1.15, 0.01, 0.12, -0.03, 0.02, 0.005],
}
# MAPX c0..c7, MAPY d0..d5, factor, unused (gopro_warp.rs:9-14) — a mild superview-like warp
GOPRO_WARP_PARAMS = [1.21, -1.27, 1.7, 0.1, 0.0, 0.0, 0.0, 0.05, 0.94, 0.44, -0.7, -0.35, 1.1, 0.35, 1.3333, 0.0]


def base_kernel_params(width, height, out_width=None, out_height=None, pixel_type="RGBA8", stride=None, out_stride=None,
                       lens="opencv_fisheye", digital_lens=None, interpolation="Bilinear", fov=1.0):
    """KernelParams as produced by FrameTransform::at_timestamp (frame_transform.rs:322-340) + get_frame_transform_at
    (stabilization/mod.rs:253-326) for host buffers without rect/rotation, defaults of stabilization_params.rs:128-192."""
    out_width = out_width or width
    out_height = out_height or height
    _, count, sdt = abi.PIXEL_TYPES[pixel_type]
    bpp = count * np.dtype(sdt).itemsize
    stride = stride or (width * bpp + 255) // 256 * 256
    out_stride = out_stride or (out_width * bpp + 255) // 256 * 256
    p = abi.KernelParams()
    p.width, p.height, p.stride = width, height, stride
    p.output_width, p.output_height, p.output_stride = out_width, out_height, out_stride
    p.matrix_count = 1
    p.interpolation = abi.INTERP[interpolation]
    if p.interpolation > 8:                          # EWA CubicBC coefficients, stabilization/mod.rs:279-295 (f32 arithmetic)
        f = np.float32
        b, c = {10: (0.2620145, 0.3689927), 11: (0.3782157, 0.3108921), 12: (0.3333333, 0.3333333), 13: (0.0, 0.5)}[p.interpolation]
        b, c = f(b), f(c)
        p.ewa_coeffs_p[:] = [float((f(6.0) - f(2.0) * b) / f(6.0)), 0.0, float((f(-18.0) + f(12.0) * b + f(6.0) * c) / f(6.0)),
                             float((f(12.0) - f(9.0) * b - f(6.0) * c) / f(6.0))]
        p.ewa_coeffs_q[:] = [float((f(8.0) * b + f(24.0) * c) / f(6.0)), float((f(-12.0) * b - f(48.0) * c) / f(6.0)),
                             float((f(6.0) * b + f(30.0) * c) / f(6.0)), float((f(-1.0) * b - f(6.0) * c) / f(6.0))]
    p.background_mode = 0
    p.flags = abi.FLAG_HAS_DIGITAL_LENS if digital_lens else 0
    p.bytes_per_pixel = bpp
    p.pix_element_count = count
    p.background[:] = [0.0, 0.0, 0.0, 0.0]
    fx = 0.5 * width
    p.f[:] = [fx, fx]
    p.c[:] = [width / 2.0, height / 2.0]
    k = list(LENS_COEFFS[lens]) + [0.0] * 12
    p.k[:] = k[:12]
    p.fov = fov * (width / max(out_width, 1))            # get_fov: fov *= width / output_width  (frame_transform.rs:56)
    p.r_limit = 0.0
    p.lens_correction_amount = 1.0
    p.input_vertical_stretch = 1.0
    p.input_horizontal_stretch = 1.0
    p.background_margin = 0.0
    p.background_margin_feather = 0.0
    p.canvas_scale = 1.0
    p.light_refraction_coefficient = 1.0
    p.source_rect[:] = [0, 0, width, height]
    p.output_rect[:] = [0, 0, out_width, out_height]
    if digital_lens == "gopro_warp":
        p.digital_lens_params[:] = GOPRO_WARP_PARAMS
    elif digital_lens == "digital_stretch":
        p.digital_lens_params[:] = [1.1, 0.95] + [0.0] * 14
    maxv = {"u1": 255.0, "u2": 65535.0}.get(sdt)
    p.max_pixel_value = maxv if maxv else 1.0                     # T::default_max_value().unwrap_or(1.0)
    p.pixel_value_limit = maxv if maxv else float(np.finfo(np.float32).max)
    p.distortion_model = abi.LENS[lens]
    p.digital_lens = abi.LENS[digital_lens] if digital_lens else 0
    p.safe_area_rect[:] = [0.0, 0.0, float(out_width), float(out_height)]
    return p


def synthetic_camera_stab(n_frames, width, height, n_points=32, seed=7):
    """CameraStabData per frame (gyro_source/file_metadata.rs:41-48) for config 4: a 6000 x 4000 sensor read through a
    (500, 300, 5000, 3400) crop, 8.4 um pixel pitch (stored x1000), IBIS (x, y, roll in millidegrees) and OIS (x, y) as Catmull-Rom
    control points over the sensor rows — +-3 px / +-0.2 degrees / +-1 px at the frame's scale, different for every frame."""
    rng = np.random.Generator(np.random.PCG64(seed))
    crop = (500.0, 300.0, 5000.0, 3400.0); pitch = (8400, 8400)
    sx = width / crop[2] / pitch[0]; sy = height / crop[3] / pitch[1]
    out = []
    for f in range(n_frames):
        pos = np.linspace(200.0, 3800.0, n_points)
        ph = rng.uniform(0, 2 * math.pi, 4)
        ibis = np.stack([3.0 / sx * np.sin(pos / 600.0 + ph[0]), -3.0 / sy * np.cos(pos / 800.0 + ph[1]), 200.0 * np.sin(pos / 1100.0 + ph[2])], axis=1)
        ois = np.stack([1.0 / sx * np.sin(pos / 350.0 + ph[3]), -1.0 / sy * np.cos(pos / 420.0 + ph[0]), np.zeros_like(pos)], axis=1)
        out.append(dict(offset=0.0, sensor_size=(6000, 4000), crop_area=crop, pixel_pitch=pitch, ibis=(pos, ibis), ois=(pos, ois)))
    return out


# ------------------------------------------------------------------------------------------ mesh (config 4)


def synthetic_mesh(width, height, amp=4.0, n=9, with_fpd=False):
    """9x9 mesh with a smooth +-amp px perturbation, laid out like sony.rs:483-511:
    header(9) | n*n (x,y) pairs | per-row cubic coefficient blocks for x then y | optional focal-plane block."""
    size = (float(width), float(height))
    xs = np.linspace(0.0, size[0], n); ys = np.linspace(0.0, size[1], n)
    pts = []
    for j in range(n):
        for i in range(n):
            dx = amp * math.sin(math.pi * i / (n - 1)) * math.cos(2.0 * math.pi * j / (n - 1))
            dy = amp * math.cos(1.5 * math.pi * i / (n - 1)) * math.sin(math.pi * j / (n - 1))
            pts += [xs[i] + dx, ys[j] + dy]
    mesh = [0.0, float(n), float(n), size[0], size[1], 0.0, 0.0, size[0], size[1]] + pts

    def coeffs(vals, sz):                     # splines.rs:100-124
        nn = len(vals); h = sz / (nn - 1); inv_h = 1.0 / h
        a = list(vals); alpha = [0.0] * nn; mu = [0.0] * nn; z = [0.0] * nn
        b = [0.0] * 9; c = [0.0] * 9; d = [0.0] * 9
        for i in range(1, nn - 1):
            alpha[i] = 3.0 * inv_h * (a[i + 1] - 2.0 * a[i] + a[i - 1])
        for i in range(1, nn - 1):
            mu[i] = 1.0 / (4.0 - mu[i - 1]); z[i] = (alpha[i] * inv_h - z[i - 1]) * mu[i]
        for j in range(nn - 2, -1, -1):
            c[j] = z[j] - mu[j] * c[j + 1]
            b[j] = (a[j + 1] - a[j]) * inv_h - (h / 3.0) * (c[j + 1] + 2.0 * c[j])
            d[j] = (c[j + 1] - c[j]) * (1.0 / (3.0 * h))
        a9 = a + [0.0] * (9 - nn)
        return a9, b, c, d

    for off in (0, 1):
        for j in range(n):
            vals = [mesh[9 + (j * n + i) * 2 + off] for i in range(n)]
            a, b, c, d = coeffs(vals, size[0])
            mesh += a + b + c + d
    mesh[0] = float(len(mesh))
    if with_fpd:
        fpd = [1.0, 0.0, 0.0, 0.0] + [v for i in range(8) for v in (0.002 * math.sin(i), 0.001 * math.cos(i))]
        mesh += fpd
    return np.asarray(mesh, dtype=np.float32)
