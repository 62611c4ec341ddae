"""Second, independent restatement of the adaptive-zoom companion — TEST INFRASTRUCTURE ONLY.

  at_timestamp_for_points   <- FrameTransform::at_timestamp_for_points    src/core/stabilization/frame_transform.rs:352-410
  undistort_points          <- undistort_points (every lens model and digital lens, IBIS / OIS shifts, distorting mesh + focal-plane distortion)
                                                                           src/core/stabilization/cpu_undistort.rs:652-858
  find_fov                  <- FovIterative::find_fov / nearest_edge / points_around_rect / interpolate_points
                                                                           src/core/zooming/fov_iterative.rs:76-200

Written from the Rust text in numpy scalars; the C oracle (oracle/gf_oracle.c, gf_oracle_find_fov) and the CUDA kernels
(gyroflow_b200/csrc/zoom_kernel.cu) are checked against it in tests/test_zoom.py and tests/test_point_matrix.py.  The rotations come
from numpy's f64 slerp / matrix products (tests/np_producer.py), which round like the oracle's on the host: the two agree bit for bit.
"""
import math

import numpy as np

from gyroflow_b200.synth import q_mul, q_inv
from tests import np_producer
from tests import np_restatement as npr
from tests.np_restatement import F, sqrtf


def get_fov(c, frame, use_fovs):                                                  # frame_transform.rs:52-58 (no Fov keyframe here)
    fov_scale = c.fov_scale + (1.0 if (c.fov_overview and use_fovs) else 0.0)
    if use_fovs:
        fovs = [c.fovs[i] for i in range(c.n_fovs)]
        f = fovs[frame] if frame < len(fovs) else (fovs[-1] if len(fovs) > 1 else 1.0)
        fov = f * fov_scale
    else:
        fov = 1.0
    fov = max(fov, 0.001)
    return fov * c.width / max(c.output_width, 1)


def point_shifts(cp, pts, stab):                                                   # frame_transform.rs:412-431 (IBIS / OIS shift of every point)
    c = cp.c
    cx, cy, cw, ch = [float(np.float32(v)) for v in stab["crop_area"]]
    pp = stab["pixel_pitch"]
    sc = (c.width / cw / float(pp[0]), c.height / ch / float(pp[1]))               # no framebuffer sign here, unlike at_timestamp
    out = []
    z = np.zeros(3)
    for (_x, y) in pts:
        ys = (float(y) - 0.0) * ((cy + ch) - cy) / (float(c.height) - 0.0) + cy    # map_coord in f64
        sv = np_producer.catmull_rom(np.asarray(stab["ibis"][0], float), np.asarray(stab["ibis"][1], float), ys + stab["offset"])
        ov = np_producer.catmull_rom(np.asarray(stab["ois"][0], float), np.asarray(stab["ois"][1], float), ys + stab["offset"])
        sv = z if sv is None else sv; ov = z if ov is None else ov
        ra = sv[2] / 1000.0
        out.append((F(sv[0] * sc[0]), F(sv[1] * sc[1]), F(ra * (math.pi / 180.0)), F(ov[0] * sc[0]), F(ov[1] * sc[1])))
    return out


def at_timestamp_for_points(cp, points, timestamp_ms, frame, use_fovs, stab=None):  # frame_transform.rs:352-438
    c = cp.c
    K = np.array(list(c.camera_matrix), dtype=np.float64).reshape(3, 3)
    fov = get_fov(c, frame, use_fovs)
    hr = c.input_horizontal_stretch if c.input_horizontal_stretch > 0.01 else 1.0  # get_new_k :37-51
    new_k = K.copy()
    new_k[0, 0] = new_k[0, 0] * (1.0 / hr) / fov; new_k[1, 1] = new_k[1, 1] * (1.0 / hr) / fov
    new_k[0, 2] = c.output_width / 2.0; new_k[1, 2] = c.output_height / 2.0
    frt = abs(c.frame_readout_time)                                                # get_frame_readout_time(can_invert = false) :21-36
    if c.readout_inverted: frt *= -1.0
    n = c.width if c.readout_horizontal else c.height
    row_readout_time = frt / n
    start_ts = timestamp_ms - frt / 2.0
    a = c.video_rotation * (math.pi / 180.0)
    image_rotation = np.array([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]])
    org = type("T", (), dict(ts=cp._ots, q=cp._oq))
    sm = type("T", (), dict(ts=cp._sts, q=cp._sq))
    quat1 = q_inv(np_producer.quat_at_timestamp(org, timestamp_ms)[0])
    sq1 = np_producer.quat_at_timestamp(sm, timestamp_ms)[0]
    pts = points if abs(frt) > 0.0 else [(0.0, 0.0)]
    rotations = []
    for (x, y) in pts:
        qt = start_ts + row_readout_time * float(x if c.readout_horizontal else y) if abs(frt) > 0.0 else start_ts
        quat = q_mul(q_mul(sq1[None, :], quat1[None, :]), np_producer.quat_at_timestamp(org, qt))[0]
        r = image_rotation @ np_producer.q_to_matrix(quat)
        r[0, 1] *= -1.0; r[0, 2] *= -1.0; r[1, 0] *= -1.0; r[2, 0] *= -1.0
        if c.suppress_rotation:
            r = np.eye(3)
        rotations.append(new_k @ r)
    shifts = point_shifts(cp, pts, stab) if stab is not None else None            # one entry per element of points_iter: a single one when RS is off
    if c.suppress_rotation and c.frame_readout_time == 0.0:                        # :432-434
        shifts = None
    return K, rotations, fov, shifts


def _refract(px, py, lrc):                                                         # cpu_undistort.rs:767-776
    if lrc != F(1.0) and lrc > 0:
        r = sqrtf(px * px + py * py)
        if r != 0:
            sin_theta_d = (r / sqrtf(F(1.0) + r * r)) / lrc
            r_d = sin_theta_d / sqrtf(F(1.0) - sin_theta_d * sin_theta_d)
            fac = r_d / r
            return px * fac, py * fac
    return px, py


class _KP:                                                                         # the KernelParams undistort_points builds (:671-683)
    pass


def _point_mesh(x, y, c, mesh):                                                   # cpu_undistort.rs:712-746 (mesh: list of f64)
    fw, fh = F(c.width), F(c.height)
    ox, oy, cw, ch = F(mesh[5]), F(mesh[6]), F(mesh[7]), F(mesh[8])
    mc = npr.map_coord
    o = int(mesh[0]) if mesh[0] > 0.0 else 0
    if mesh[0] > 0.0 and o < len(mesh) and mesh[o] > 0.0:                          # FocalPlaneDistortion: ADDED on this path
        stblz_grid = mesh[4] / 8.0
        x = mc(x, 0.0, fw, ox, ox + cw); y = mc(y, 0.0, fh, oy, oy + ch)
        q = math.floor(float(y) / stblz_grid)
        idx = int(min(max(q, 0.0), 7.0)) if not math.isnan(q) else 0
        delta = float(y) - stblz_grid * idx
        x = x + F(mesh[o + 4 + idx * 2 + 0] * delta); y = y + F(mesh[o + 4 + idx * 2 + 1] * delta)
        for j in range(idx):
            x = x + F(mesh[o + 4 + j * 2 + 0] * stblz_grid); y = y + F(mesh[o + 4 + j * 2 + 1] * stblz_grid)
        x = mc(x, ox, ox + cw, 0.0, fw); y = mc(y, oy, oy + ch, 0.0, fh)
    if mesh[0] > 10.0:
        x = mc(x, 0.0, fw, ox, ox + cw); y = mc(y, 0.0, fh, oy, oy + ch)
        nx, ny = npr.interpolate_mesh(float(x), float(y), (mesh[3], mesh[4]), mesh)
        x = mc(F(nx), ox, ox + cw, 0.0, fw); y = mc(F(ny), oy, oy + ch, 0.0, fh)
    return x, y


def undistort_points(cp, points, K, rotations, lens_correction_amount, fov, lens="opencv_fisheye", digital=None, shifts=None, mesh=None):   # cpu_undistort.rs:652-858 (no mesh / IBIS shifts)
    c = cp.c
    kp = _KP()
    kp.width, kp.height, kp.output_width, kp.output_height = c.width, c.height, c.output_width, c.output_height
    kp.digital_lens_params = [F(v) for v in list(c.digital_lens_params)]
    und, dist = npr.UNDISTORT[lens], npr.DISTORT[lens]
    dund = npr.DIGITAL_UNDISTORT[digital] if digital else None
    ddist = npr.DIGITAL[digital] if digital else None
    fx, fy, cx, cy = F(K[0, 0]), F(K[1, 1]), F(K[0, 2]), F(K[1, 2])
    k = [F(v) for v in list(c.distortion_coeffs)]
    lrc = F(c.light_refraction_coefficient)
    lc = None
    if lens_correction_amount < 1.0:                                               # :686-694
        out_c = (F(c.output_width) / F(2.0), F(c.output_height) / F(2.0))
        amount = F(lens_correction_amount)
        factor = max(F(1.0) - amount, F(0.001))
        out_f = (fx / F(fov) / factor, fy / F(fov) / factor)
        lc = (out_c, amount, factor, out_f)
    out = []
    for index, (x, y) in enumerate(points):
        x, y = F(x), F(y)
        if c.input_horizontal_stretch > 0.001: x = x * F(c.input_horizontal_stretch)      # :702-703
        if c.input_vertical_stretch > 0.001: y = y * F(c.input_vertical_stretch)
        if dund is not None:                                                       # :705-710
            x, y = dund(x, y, kp)
        if mesh is not None and len(mesh) > 9:
            x, y = _point_mesh(x, y, c, mesh)
        if shifts is not None and index < len(shifts):                             # :748-757 (sic: y is rotated with the UPDATED x)
            sh = shifts[index]
            cos_a = npr.cosf(sh[2]); sin_a = npr.sinf(sh[2])
            x = x - cx - sh[3] + sh[0]
            y = y - cy - sh[4] + sh[1]
            x = cos_a * x - sin_a * y + cx
            y = sin_a * x + cos_a * y + cy
        pwx, pwy = (x - cx) / fx, (y - cy) / fy                                    # :760
        rot = np.asarray(rotations[index] if index < len(rotations) else rotations[0], dtype=np.float64).astype(np.float32)
        pt = und(pwx, pwy, k)
        if pt is None:
            out.append((F(-1000000.0), F(-1000000.0)))
            continue
        px, py = _refract(pt[0], pt[1], lrc)
        pr = [rot[i, 0] * px + rot[i, 1] * py + rot[i, 2] * F(1.0) for i in range(3)]   # rot * (x, y, 1) in f32
        px, py = pr[0] / pr[2], pr[1] / pr[2]
        if lc is not None:                                                         # :782-852: solve amount*o + factor*R(o) = pt by Newton
            out_c, amount, factor, out_f = lc

            def r_of(ox, oy):
                if dund is not None:                                               # un-zoom -> digital warp -> re-zoom (:795-801)
                    uzx, uzy = (ox - out_c[0]) * F(fov) + out_c[0], (oy - out_c[1]) * F(fov) + out_c[1]
                    d = dund(uzx, uzy, kp)
                    ox, oy = (d[0] - out_c[0]) / F(fov) + out_c[0], (d[1] - out_c[1]) / F(fov) + out_c[1]
                nx, ny = (ox - out_c[0]) / out_f[0], (oy - out_c[1]) / out_f[1]
                d = und(nx, ny, k)
                if d is not None: nx, ny = d
                nx, ny = _refract(nx, ny, lrc)
                return (nx * out_f[0]) + out_c[0], (ny * out_f[1]) + out_c[1]

            nx, ny = (px - out_c[0]) / out_f[0], (py - out_c[1]) / out_f[1]
            dx, dy = dist(nx, ny, F(1.0), k)
            p2x, p2y = (dx * out_f[0]) + out_c[0], (dy * out_f[1]) + out_c[1]
            if ddist is not None:                                                  # :826-830
                uzx, uzy = (p2x - out_c[0]) * F(fov) + out_c[0], (p2y - out_c[1]) * F(fov) + out_c[1]
                dd = ddist(uzx, uzy, kp)
                p2x, p2y = (dd[0] - out_c[0]) / F(fov) + out_c[0], (dd[1] - out_c[1]) / F(fov) + out_c[1]
            if math.isfinite(float(p2x)) and math.isfinite(float(p2y)):
                ox, oy = p2x * factor + px * amount, p2y * factor + py * amount
            else:
                ox, oy = px, py
            for _ in range(10):
                rx, ry = r_of(ox, oy)
                g0, g1 = amount * ox + factor * rx - px, amount * oy + factor * ry - py
                if abs(g0) < F(0.02) and abs(g1) < F(0.02): break
                eps = F(1.0)
                rxx, rxy = r_of(ox + eps, oy)
                ryx, ryy = r_of(ox, oy + eps)
                j11 = amount + factor * (rxx - rx) / eps; j21 = factor * (rxy - ry) / eps
                j12 = factor * (ryx - rx) / eps;          j22 = amount + factor * (ryy - ry) / eps
                det = j11 * j22 - j12 * j21
                if not math.isfinite(float(det)) or abs(det) < F(1e-9): break
                ddx = (j22 * g0 - j12 * g1) / det
                ddy = (-j21 * g0 + j11 * g1) / det
                if not math.isfinite(float(ddx)) or not math.isfinite(float(ddy)): break
                ox, oy = ox - ddx, oy - ddy
            px, py = ox, oy
        out.append((px, py))
    return out


def undistort_points_with_rolling_shutter(cp, points, timestamp_ms, frame, lens_correction_amount, use_fovs=False, lens="opencv_fisheye", digital=None, stab=None, mesh=None):   # :636-641
    """stab: the CameraStabData dict of this frame (as given to backend.ComputeParams(camera_stab=[...])) or None."""
    K, rotations, fov, shifts = at_timestamp_for_points(cp, points, timestamp_ms, frame, use_fovs, stab)
    return undistort_points(cp, points, K, rotations, lens_correction_amount, fov, lens, digital, shifts, mesh)


def points_around_rect(w, h, w_div, h_div, margin):                                # fov_iterative.rs:154-177
    w, h, margin = F(w), F(h), F(margin)
    w = w - margin * F(2.0); h = h - margin * F(2.0)
    wcnt, hcnt = max(w_div, 2) - 1, max(h_div, 2) - 1
    wstep, hstep = w / F(wcnt), h / F(hcnt)
    pts = [(F(i) * wstep, F(0.0)) for i in range(wcnt)] + [(w, F(i) * hstep) for i in range(hcnt)] + \
          [(F(wcnt - i) * wstep, h) for i in range(wcnt)] + [(F(0.0), F(hcnt - i) * hstep) for i in range(hcnt)]
    return [(x + margin, y + margin) for x, y in pts]


def interpolate_points(pts, steps):                                                # fov_iterative.rs:182-192
    d = steps + 1
    new_len = d * len(pts) - steps
    out = []
    for i in range(new_len):
        idx1 = i // d
        idx2 = min(idx1 + 1, len(pts) - 1)
        f = F(i % d) / F(d)
        out.append((pts[idx1][0] + f * (pts[idx2][0] - pts[idx1][0]), pts[idx1][1] + f * (pts[idx2][1] - pts[idx1][1])))
    return out


def nearest_edge(polygon, center, initial, inv_aspect):                            # fov_iterative.rs:136-151
    idx, mp = None, initial
    for i, (x, y) in enumerate(polygon):
        ap = (abs(x - center[0]), abs(y - center[1]))
        if ap[0] < mp[0] and ap[1] < mp[1]:
            if ap[1] > ap[0] * inv_aspect:
                idx, mp = i, (ap[1] / inv_aspect, ap[1])
            else:
                idx, mp = i, (ap[0], ap[0] * inv_aspect)
    return idx, mp


def find_fov(cp, org_output_size, timestamp_ms, frame, margin=2.0, lens="opencv_fisheye", digital=None, stab=None):               # FovIterative::new :76-89 + find_fov :91-134
    """`cp` must already carry the calculate_fovs adjustments (zooming/mod.rs:41-49): fov_scale 1, no fovs, output size = input size."""
    c = cp.c
    ratio = F(c.width) / F(max(org_output_size[0], 1))
    input_dim = (F(c.width), F(c.height))
    output_dim = (F(org_output_size[0]) * ratio, F(org_output_size[1]) * ratio)
    inv_aspect = output_dim[1] / output_dim[0]
    rect = points_around_rect(input_dim[0], input_dim[1], 31, 31, margin)
    center = (input_dim[0] / F(2.0), input_dim[1] / F(2.0))
    zx, zy, lca = c.adaptive_zoom_center_offset[0], c.adaptive_zoom_center_offset[1], c.lens_correction_amount

    def shifted(pts):
        poly = undistort_points_with_rolling_shutter(cp, pts, timestamp_ms, frame, lca, False, lens, digital, stab)
        return [(x - F(zx) * input_dim[0], y - F(zy) * input_dim[1]) for x, y in poly]

    polygon = shifted(rect)
    nearest = (None, (F(1000000.0), F(1000000.0) * inv_aspect))
    for _ in range(1, 5):
        nearest = nearest_edge(polygon, center, nearest[1], inv_aspect)
        if nearest[0] is None:
            break
        n = len(rect)
        idx = nearest[0]
        # `idx.overflowing_sub(1).0 % len`: usize wrap-around, (2^64 - 1) % len for idx == 0
        relevant = [rect[((idx - 1) % (1 << 64)) % n], rect[idx], rect[(idx + 1) % n]]
        polygon = shifted(interpolate_points(relevant, 30))
        nearest = nearest_edge(polygon, center, nearest[1], inv_aspect)
    return float(nearest[1][0] * F(2.0) / output_dim[0])


# ---- zoom_dynamic::compute, static-window branch — src/core/zooming/zoom_dynamic.rs:56-76 and helpers :80-124, :167-191 (Python floats = f64) ----
def zoom_dynamic(fov_values, window_s, fps, method):
    """method 0: GaussianFilter (rolling minimum, then a normalised Gaussian over `frames` samples); 1: EnvelopeFollower (two passes)."""
    v = [float(x) for x in fov_values]

    def pad_edge(arr, n):                                                         # :111-124
        return [arr[0]] * n + list(arr) + [arr[-1]] * n

    def envelope_follower(a, alpha):                                              # :167-191 with a constant alpha
        q = a[-1]
        rev = []
        for x in reversed(a):
            q = min(x, x * alpha + q * (1.0 - alpha))
            rev.append(q)                                                         # rev[0] belongs to the LAST sample
        q = rev[-1]
        out = []
        for x in reversed(rev):
            q = min(x, x * alpha + q * (1.0 - alpha))
            out.append(q)
        return out

    if method == 0:
        frames = int(math.floor(window_s * fps))                                  # get_frames_per_window :80-86
        if frames % 2 == 0:
            frames += 1
        padded = pad_edge(v, frames // 2)
        fov_min = [min(padded[i:i + frames]) for i in range(len(padded) - frames + 1)]          # min_rolling :88-92
        padded = pad_edge(fov_min, frames // 2)
        std = frames / 6.0
        sig2 = 2.0 * std ** 2                                                     # gaussian_window :100-103 (powi(2) == x * x)
        half = frames // 2
        w = [math.exp(-float(x * x) / sig2) for x in range(-half, half + 1)]
        s = 0.0
        for t in w: s += t
        w = [t / s for t in w]                                                    # gaussian_window_normalized :105-110
        out = []
        for i in range(len(padded) - frames + 1):                                 # convolve :94-98: left-to-right sum of products
            acc = 0.0
            for x, y in zip(padded[i:i + frames], w): acc += x * y
            out.append(acc)
        return out
    first = 1.0 - math.exp(-(1.0 / fps) / window_s)                               # :69-73
    second = 1.0 - math.exp(-(1.0 / fps) / 0.2)
    return envelope_follower(envelope_follower(v, first), second)
