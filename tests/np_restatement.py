"""An independent second restatement of the north-star path, written from the reference text in a different language
(Python scalars of numpy.float32) than the C oracle, to cross-check it: every physical lens model (opencv_fisheye,
opencv_standard, poly3, poly5, ptlens, insta360, sony, generic_polynomial, gopro), every digital lens (gopro_superview,
gopro6_superview, gopro_hyperview, gopro_warp, digital_stretch), vertical rolling shutter, bilinear / bicubic / Lanczos4
sampling, background modes 0-2, r_limit, light refraction, IBIS / OIS rows, input rotation and stretch, horizontal rolling shutter,
the f64 mesh correction (bivariate spline, splines.rs:100-176 / sony.rs:557-563) and focal-plane distortion, the EWA CubicBC resampler,
background mode 3 (margin with feather), fix-colour-range and fill-with-background, and the lens-correction blend with every model's
undistort_point (physical and digital),
on 8-bit, 16-bit and f32 pixels (cpu_undistort.rs:133-228, :262-418, :421-517, :519-633; distortion_models/*.rs distort_point;
gyro_source/splines.rs; util.rs:144-147; pixel_formats.rs conversions).
With it every lens formula and every optional stage of the oracle has two independent transcriptions.

TEST INFRASTRUCTURE ONLY.  numpy.float32 arithmetic is IEEE single precision without contraction; atan goes to the same
libm `atanf` Rust's std calls (numpy's own arctan may differ in the last ulp)."""
import ctypes
import ctypes.util
import math

import numpy as np

F = np.float32
_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.atanf.restype = ctypes.c_float
_libm.atanf.argtypes = [ctypes.c_float]
_libm.sqrtf.restype = ctypes.c_float
_libm.sqrtf.argtypes = [ctypes.c_float]
_libm.tanf.restype = ctypes.c_float
_libm.tanf.argtypes = [ctypes.c_float]
_libm.sinf.restype = ctypes.c_float
_libm.sinf.argtypes = [ctypes.c_float]
_libm.cosf.restype = ctypes.c_float
_libm.cosf.argtypes = [ctypes.c_float]


def atanf(x):
    return F(_libm.atanf(float(x)))


def sinf(x):
    return F(_libm.sinf(float(x)))


def cosf(x):
    return F(_libm.cosf(float(x)))


def tanf(x):
    return F(_libm.tanf(float(x)))


def sqrtf(x):
    return F(_libm.sqrtf(float(x)))          # IEEE correctly rounded, same as f32::sqrt


def round_half_away(x):                      # f32::round
    x = float(x)
    if math.isnan(x) or math.isinf(x):
        return F(x)
    return F(math.copysign(math.floor(abs(x) + 0.5), x)) if abs(x) < 2 ** 23 else F(x)


def as_i32(x):                               # Rust `as i32`: truncate, saturate, NaN -> 0
    x = float(x)
    if math.isnan(x):
        return 0
    if x >= 2147483647.0:
        return 2147483647
    if x <= -2147483648.0:
        return -2147483648
    return int(x)


def map_coord(x, in_min, in_max, out_min, out_max):      # util.rs:144-147
    return (F(x) - F(in_min)) * (F(out_max) - F(out_min)) / (F(in_max) - F(in_min)) + F(out_min)


def fisheye_distort(x, y, z, k):             # opencv_fisheye.rs:72-93
    x = x / z; y = y / z
    if k[0] == 0 and k[1] == 0 and k[2] == 0 and k[3] == 0:         # :75
        return x, y
    r = sqrtf(x * x + y * y)
    theta = atanf(r)
    theta2 = theta * theta; theta4 = theta2 * theta2; theta6 = theta4 * theta2; theta8 = theta4 * theta4
    theta_d = theta * (F(1.0) + k[0] * theta2 + k[1] * theta4 + k[2] * theta6 + k[3] * theta8)
    scale = F(1.0) if r == F(0.0) else theta_d / r
    return x * scale, y * scale


def standard_distort(x, y, z, k):            # opencv_standard.rs:32-48
    x = x / z; y = y / z
    r2 = x * x + y * y; r4 = r2 * r2; r6 = r4 * r2
    a1 = F(2.0) * x * y; a2 = r2 + F(2.0) * x * x; a3 = r2 + F(2.0) * y * y
    cdist = F(1.0) + k[0] * r2 + k[1] * r4 + k[4] * r6
    icdist2 = F(1.0) / (F(1.0) + k[5] * r2 + k[6] * r4 + k[7] * r6)
    return (x * cdist * icdist2 + k[2] * a1 + k[3] * a2 + k[8] * r2 + k[9] * r4,
            y * cdist * icdist2 + k[2] * a3 + k[3] * a1 + k[10] * r2 + k[11] * r4)


def poly3_distort(x, y, z, k):               # poly3.rs:54-63
    x = x / z; y = y / z
    poly2 = k[0] * (x * x + y * y) + F(1.0)
    return x * poly2, y * poly2


def poly5_distort(x, y, z, k):               # poly5.rs:43-53
    x = x / z; y = y / z
    ru2 = x * x + y * y
    poly4 = F(1.0) + k[0] * ru2 + k[1] * ru2 * ru2
    return x * poly4, y * poly4


def ptlens_distort(x, y, z, k):              # ptlens.rs:42-53
    x = x / z; y = y / z
    ru2 = x * x + y * y
    r = sqrtf(ru2)
    poly3 = k[0] * ru2 * r + k[1] * ru2 + k[2] * r + F(1.0)
    return x * poly3, y * poly3


def sony_distort(x, y, z, k):                # sony.rs:65-89
    x = x / z; y = y / z
    if k[0] == 0 and k[1] == 0 and k[2] == 0 and k[3] == 0:
        return x, y
    r = sqrtf(x * x + y * y)
    theta = atanf(r)
    theta2 = theta * theta; theta3 = theta2 * theta; theta4 = theta2 * theta2; theta5 = theta2 * theta3; theta6 = theta3 * theta3
    theta_d = theta * k[0] + theta2 * k[1] + theta3 * k[2] + theta4 * k[3] + theta5 * k[4] + theta6 * k[5]
    scale = F(1.0) if r == F(0.0) else theta_d / r
    return x * scale, y * scale


def insta360_distort(x, y, z, k):            # insta360.rs:27-48
    k1, k2, k3, p1, p2, xi = k[0], k[1], k[2], k[3], k[4], k[5]
    ln = sqrtf(x * x + y * y + z * z)
    x = (x / ln) / ((z / ln) + xi)
    y = (y / ln) / ((z / ln) + xi)
    r2 = x * x + y * y; r4 = r2 * r2; r6 = r4 * r2
    return (x * (F(1.0) + k1 * r2 + k2 * r4 + k3 * r6) + F(2.0) * p1 * x * y + p2 * (r2 + F(2.0) * x * x),
            y * (F(1.0) + k1 * r2 + k2 * r4 + k3 * r6) + F(2.0) * p2 * x * y + p1 * (r2 + F(2.0) * y * y))


def generic_polynomial_distort(x, y, z, k):  # generic_polynomial.rs:83-122
    x = x / z; y = y / z
    if all(k[i] == 0 for i in range(12)):
        return x, y
    r = sqrtf(x * x + y * y)
    t = atanf(r)
    t2 = t * t; t3 = t2 * t; t4 = t2 * t2; t5 = t2 * t3; t6 = t3 * t3; t7 = t3 * t4; t8 = t4 * t4; t9 = t4 * t5
    t10 = t5 * t5; t11 = t5 * t6; t12 = t6 * t6
    theta_d = (t * k[0] + t2 * k[1] + t3 * k[2] + t4 * k[3] + t5 * k[4] + t6 * k[5] + t7 * k[6] + t8 * k[7] + t9 * k[8]
               + t10 * k[9] + t11 * k[10] + t12 * k[11])
    scale = F(1.0) if r == F(0.0) else theta_d / r
    return x * scale, y * scale


def _gopro_poly_eval(p, k):                  # gopro.rs:19-21
    return k[0] + p * (k[1] + p * (k[2] + p * (k[3] + p * (k[4] + p * (k[5] + p * k[6])))))


def _gopro_poly_deriv(p, k):                 # gopro.rs:22-24
    return k[1] + p * (F(2.0) * k[2] + p * (F(3.0) * k[3] + p * (F(4.0) * k[4] + p * (F(5.0) * k[5] + p * (F(6.0) * k[6])))))


def gopro_distort(x, y, z, k):               # gopro.rs:56-72 with poly_invert :26-36
    px, py = x / z, y / z
    if k[1] == 0:
        return px, py
    r = sqrtf(px * px + py * py)
    TMAX = F(1.5533)
    tt = tanf(TMAX)
    theta = atanf(r) if r < tt else TMAX + (r - tt) / (F(1.0) + tt * tt)
    p = (theta - k[0]) / k[1]
    for _ in range(10):
        d = _gopro_poly_deriv(p, k)
        if abs(d) < F(1e-12):
            break
        fix = (_gopro_poly_eval(p, k) - theta) / d
        p = p - fix
        if abs(fix) < F(1e-7):
            break
    r_norm = k[1] * p
    scale = F(1.0) if r < F(1e-9) else r_norm / r
    return px * scale, py * scale


DISTORT = {"opencv_fisheye": fisheye_distort, "opencv_standard": standard_distort, "poly3": poly3_distort, "poly5": poly5_distort,
           "ptlens": ptlens_distort, "sony": sony_distort, "insta360": insta360_distort, "generic_polynomial": generic_polynomial_distort,
           "gopro": gopro_distort}


# ---- digital lenses: distort_point (wide -> recorded), cpu_undistort.rs:216-220 ------------------------------------------------
def _superview(ux, uy):                      # gopro_superview.rs:12-19
    x2 = ux * ux; y2 = uy * uy
    return (ux * (F(1.2100393) + x2 * (F(-1.2758402) + x2 * F(1.7751845))),
            uy * (F(0.9364505) + (F(0.4465308) - F(0.7683315) * y2) * y2 + (F(-0.3574087) + F(1.1584653) * y2 + F(0.3529348) * x2) * x2))


def _superview6(ux, uy):                     # gopro6_superview.rs:12-17
    ux = ux * (F(1.0) - F(0.48) * abs(ux))
    ux = ux * (F(0.943396) * (F(1.0) + F(0.157895) * abs(ux)))
    uy = uy * (F(0.943396) * (F(1.0) + F(0.060000) * abs(uy * F(2.0))))
    return ux, uy


def _hyperview(ux, uy):                      # gopro_hyperview.rs:10-17
    x2 = ux * ux; y2 = uy * uy
    return (ux * (F(1.5805143) + x2 * (F(-8.1668825) + x2 * (F(74.5198746) + x2 * (F(-451.5002441) + x2 * (F(1551.2922363) + x2 * (F(-2735.5422363) + x2 * F(1923.1572266))))))
                  + y2 * F(-0.1086027)),
            uy * (F(1.0238225) + y2 * F(-0.1025671) + x2 * (F(-0.2639930) + x2 * F(0.2979266))))


def _view_distort(fn, xscale):               # the distort_point shared by the three *view lenses (e.g. gopro_superview.rs:37-57)
    def distort(x, y, p):
        sw, sh = F(p.width), F(p.height)
        x = (x / sw) - F(0.5); y = (y / sh) - F(0.5)
        if xscale is not None:
            x = x * F(xscale)
        ppx, ppy = x, y
        for _ in range(12):
            dx, dy = fn(ppx, ppy)
            dx = dx - x; dy = dy - y
            if abs(dx) < F(1e-6) and abs(dy) < F(1e-6):
                break
            ppx = ppx - dx; ppy = ppy - dy
        return (ppx + F(0.5)) * sw, (ppy + F(0.5)) * sh
    return distort


def _gopro_map(ux, uy, q):                   # gopro_warp.rs:22-41
    x = min(max(ux, F(-0.5)), F(0.5)); y = min(max(uy, F(-0.5)), F(0.5))
    x2 = x * x; y2 = y * y
    poly_x = q[0] + x2 * (q[1] + x2 * (q[2] + x2 * (q[3] + x2 * (q[4] + x2 * (q[5] + x2 * q[6])))))
    return (x * (poly_x + q[7] * y2) + (ux - x),
            y * (q[8] + q[9] * y2 + q[10] * y2 * y2 + x2 * (q[11] + q[12] * y2 + q[13] * x2)) + (uy - y))


def gopro_warp_distort(x, y, p):             # gopro_warp.rs:57-94
    q = [F(v) for v in p.digital_lens_params]
    factor = q[14] if q[14] != 0 else F(1.0)
    sw, sh = F(p.width), F(p.height)
    x = (x / sw) - F(0.5); y = (y / sh) - F(0.5)
    tx, ty = x * factor, y
    ppx, ppy = x, y
    for _ in range(12):
        dx, dy = _gopro_map(ppx, ppy, q)
        dx = dx - tx; dy = dy - ty
        if abs(dx) < F(1e-6) and abs(dy) < F(1e-6):
            break
        ppx = ppx - dx; ppy = ppy - dy
    rx, ry = _gopro_map(ppx, ppy, q)
    if abs(rx - tx) > F(0.02) or abs(ry - ty) > F(0.02):
        return F(-99999.0), F(-99999.0)
    return (ppx + F(0.5)) * sw, (ppy + F(0.5)) * sh


def digital_stretch_distort(x, y, p):        # digital_stretch.rs:19-22
    return x * F(p.digital_lens_params[0]), y * F(p.digital_lens_params[1])


def fmaxf(a, b):                             # f32::max: the other operand if one is NaN
    if math.isnan(float(a)): return F(b)
    if math.isnan(float(b)): return F(a)
    return F(a) if a > b else F(b)


def fminf(a, b):                             # f32::min
    if math.isnan(float(a)): return F(b)
    if math.isnan(float(b)): return F(a)
    return F(a) if a < b else F(b)


def fisheye_undistort_point(x, y, k):        # opencv_fisheye.rs:12-66
    if k[0] == 0 and k[1] == 0 and k[2] == 0 and k[3] == 0:
        return x, y
    EPS = F(1e-6)
    PI = F(math.pi)
    theta_d = sqrtf(x * x + y * y)
    theta_d = fminf(fmaxf(theta_d, -PI), PI)
    converged = False
    theta = theta_d
    scale = F(0.0)
    if abs(theta_d) > EPS:
        theta = F(0.0)
        for _ in range(10):
            theta2 = theta * theta
            theta4 = theta2 * theta2
            theta6 = theta4 * theta2
            theta8 = theta6 * theta2
            k0_theta2 = k[0] * theta2
            k1_theta4 = k[1] * theta4
            k2_theta6 = k[2] * theta6
            k3_theta8 = k[3] * theta8
            theta_fix = (theta * (F(1.0) + k0_theta2 + k1_theta4 + k2_theta6 + k3_theta8) - theta_d) / \
                        (F(1.0) + F(3.0) * k0_theta2 + F(5.0) * k1_theta4 + F(7.0) * k2_theta6 + F(9.0) * k3_theta8)
            theta_fix = fminf(fmaxf(theta_fix, F(-0.9)), F(0.9))
            theta = theta - theta_fix
            if abs(theta_fix) < EPS:
                converged = True
                break
        scale = tanf(theta) / theta_d
    else:
        converged = True
    theta_flipped = (theta_d < 0 and theta > 0) or (theta_d > 0 and theta < 0)
    if converged and not theta_flipped:
        return x * scale, y * scale
    return None


# ---- undistort_point of the other lens models (the lens-correction blend, ST maps and the zoom companion call them) ----
NEWTON_EPS = F(0.00001)


def standard_undistort_point(x, y, k):       # opencv_standard.rs:12-31
    x0, y0 = x, y
    for _ in range(20):
        r2 = x * x + y * y
        icdist = (F(1.0) + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (F(1.0) + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2)
        if icdist < 0:
            return None
        delta_x = F(2.0) * k[2] * x * y + k[3] * (r2 + F(2.0) * x * x) + k[8] * r2 + k[9] * r2 * r2
        delta_y = k[2] * (r2 + F(2.0) * y * y) + F(2.0) * k[3] * x * y + k[10] * r2 + k[11] * r2 * r2
        x = (x0 - delta_x) * icdist
        y = (y0 - delta_y) * icdist
    return x, y


def _radial_newton(x, y, f, df):             # the loop shared by poly3.rs:14-51, poly5.rs:14-42, ptlens.rs:15-42
    rd = sqrtf(x * x + y * y)
    if rd == 0:
        return None
    ru = rd
    for i in range(10):
        fru = f(ru, rd)
        if fru >= -NEWTON_EPS and fru < NEWTON_EPS:
            break
        if i > 5:
            return None
        ru = ru - (fru / df(ru))
    if ru < 0:
        return None
    ru = ru / rd
    return x * ru, y * ru


def poly3_undistort_point(x, y, k):          # poly3.rs:14-51
    inv_k1 = F(1.0) / k[0]
    rd = sqrtf(x * x + y * y)
    rd_div_k1 = rd * inv_k1
    return _radial_newton(x, y, lambda ru, _rd: ru * ru * ru + ru * inv_k1 - rd_div_k1, lambda ru: F(3.0) * ru * ru + inv_k1)


def poly5_undistort_point(x, y, k):          # poly5.rs:14-42
    def f(ru, rd):
        ru2 = ru * ru
        return ru * (F(1.0) + k[0] * ru2 + k[1] * ru2 * ru2) - rd

    def df(ru):
        ru2 = ru * ru
        return F(1.0) + F(3.0) * k[0] * ru2 + F(5.0) * k[1] * ru2 * ru2
    return _radial_newton(x, y, f, df)


def ptlens_undistort_point(x, y, k):         # ptlens.rs:15-42
    return _radial_newton(x, y, lambda ru, rd: ru * (k[0] * ru * ru * ru + k[1] * ru * ru + k[2] * ru + F(1.0)) - rd,
                          lambda ru: F(4.0) * k[0] * ru * ru * ru + F(3.0) * k[1] * ru * ru + F(2.0) * k[2] * ru + F(1.0))


def _theta_newton(x, y, k, n):               # sony.rs:10-61 (n = 6) and generic_polynomial.rs:18-81 (n = 12): Newton on theta * sum k_i theta^i = theta_d
    if all(k[i] == 0 for i in range(4 if n == 6 else 12)):
        return x, y
    EPS = F(1e-6)
    theta_d = sqrtf(x * x + y * y)
    converged = False
    theta = theta_d
    scale = F(0.0)
    if abs(theta_d) > EPS:
        theta = F(0.0)
        for _ in range(10):
            t2 = theta * theta; t3 = t2 * theta; t4 = t2 * t2; t5 = t2 * t3
            pw = [None, theta, t2, t3, t4, t5]
            if n == 12:
                t6 = t3 * t3; t7 = t3 * t4; t8 = t4 * t4; t9 = t4 * t5; t10 = t5 * t5; t11 = t5 * t6
                pw += [t6, t7, t8, t9, t10, t11]
            terms = [k[0]] + [k[i] * pw[i] for i in range(1, n)]
            num = terms[0]
            for t in terms[1:]: num = num + t
            den = terms[0]
            for i in range(1, n): den = den + F(i + 1) * terms[i]
            theta_fix = (theta * num - theta_d) / den
            theta = theta - theta_fix
            if abs(theta_fix) < EPS:
                converged = True
                break
        scale = tanf(theta) / theta_d
    else:
        converged = True
    flipped = (theta_d < 0 and theta > 0) or (theta_d > 0 and theta < 0)
    if converged and not flipped:
        return x * scale, y * scale
    return None


def sony_undistort_point(x, y, k):
    return _theta_newton(x, y, k, 6)


def generic_polynomial_undistort_point(x, y, k):
    return _theta_newton(x, y, k, 12)


def insta360_undistort_point(x, y, k):       # insta360.rs:10-25: fixed point on distort_point, up to 200 steps
    px, py = x, y
    for _ in range(200):
        dx, dy = insta360_distort(px, py, F(1.0), k)
        d0, d1 = dx - x, dy - y
        if abs(d0) < F(1e-6) and abs(d1) < F(1e-6):
            break
        px = px - d0; py = py - d1
    return px, py


def gopro_undistort_point(x, y, k):          # gopro.rs:40-55
    if k[1] == 0:
        return x, y
    r_norm = sqrtf(x * x + y * y)
    if r_norm < F(1e-9):
        return x, y
    p = r_norm / k[1]
    theta = _gopro_poly_eval(p, k)
    TMAX = F(1.5533)
    tt = tanf(TMAX)
    rr = tanf(theta) if theta < TMAX else tt + (theta - TMAX) * (F(1.0) + tt * tt)
    scale = rr / r_norm
    return x * scale, y * scale


UNDISTORT = {"opencv_fisheye": fisheye_undistort_point, "opencv_standard": standard_undistort_point, "poly3": poly3_undistort_point,
             "poly5": poly5_undistort_point, "ptlens": ptlens_undistort_point, "sony": sony_undistort_point, "insta360": insta360_undistort_point,
             "generic_polynomial": generic_polynomial_undistort_point, "gopro": gopro_undistort_point}


def _view_undistort(fn, xscale):             # e.g. gopro_superview.rs:23-34: the forward polynomial in normalised output coordinates
    def undistort(ux, uy, p):
        ow, oh = F(p.output_width), F(p.output_height)
        ux, uy = (ux / ow) - F(0.5), (uy / oh) - F(0.5)
        ux, uy = fn(ux, uy)
        if xscale is not None:
            ux = ux / F(xscale)
        return (ux + F(0.5)) * ow, (uy + F(0.5)) * oh
    return undistort


def gopro_warp_undistort(ux, uy, p):         # gopro_warp.rs:42-55
    q = [F(v) for v in p.digital_lens_params]
    factor = q[14] if q[14] != 0 else F(1.0)
    ow, oh = F(p.output_width), F(p.output_height)
    ux, uy = (ux / ow) - F(0.5), (uy / oh) - F(0.5)
    ux, uy = _gopro_map(ux, uy, q)
    ux = ux / factor
    return (ux + F(0.5)) * ow, (uy + F(0.5)) * oh


def digital_stretch_undistort(ux, uy, p):    # digital_stretch.rs:12-15
    return ux / F(p.digital_lens_params[0]), uy / F(p.digital_lens_params[1])


DIGITAL_UNDISTORT = {"gopro_superview": _view_undistort(_superview, 1.333333333), "gopro6_superview": _view_undistort(_superview6, None),
                     "gopro_hyperview": _view_undistort(_hyperview, 1.555555555), "gopro_warp": gopro_warp_undistort,
                     "digital_stretch": digital_stretch_undistort}


DIGITAL = {"gopro_superview": _view_distort(_superview, 1.333333333), "gopro6_superview": _view_distort(_superview6, None),
           "gopro_hyperview": _view_distort(_hyperview, 1.555555555), "gopro_warp": gopro_warp_distort, "digital_stretch": digital_stretch_distort}



# ---- f64 mesh correction: gyro_source/splines.rs:100-176 (BivariateSpline) and sony.rs:557-563 (interpolate_mesh); Python floats are IEEE doubles ----
MAX_GRID = 9


def cubic_spline_coefficients(vals, size, n):               # splines.rs:100-124 with step = 1, offset = 0
    h = size / (n - 1)
    inv_h = 1.0 / h
    three_inv_h = 3.0 * inv_h
    h_over_3 = h / 3.0
    inv_3h = 1.0 / (3.0 * h)
    a = [vals[i] for i in range(n)]
    alpha = [0.0] * MAX_GRID; mu = [0.0] * MAX_GRID; z = [0.0] * MAX_GRID
    b = [0.0] * MAX_GRID; c = [0.0] * MAX_GRID; d = [0.0] * MAX_GRID
    for i in range(1, n - 1):
        alpha[i] = three_inv_h * (a[i + 1] - 2.0 * a[i] + a[i - 1])
    for i in range(1, n - 1):
        mu[i] = 1.0 / (4.0 - mu[i - 1])
        z[i] = (alpha[i] * inv_h - z[i - 1]) * mu[i]
    c[n - 1] = 0.0
    for j in range(n - 2, -1, -1):
        c[j] = z[j] - mu[j] * c[j + 1]
        b[j] = (a[j + 1] - a[j]) * inv_h - h_over_3 * (c[j + 1] + 2.0 * c[j])
        d[j] = (c[j + 1] - c[j]) * inv_3h
    return a, b, c, d


def _as_usize(x):                                           # Rust `as usize`: truncate, saturate at 0, NaN -> 0
    if math.isnan(x) or x <= 0.0:
        return 0
    return int(min(x, 1.8446744073709552e19))


def cubic_spline_interpolate(a, b, c, d, n, x, size):       # splines.rs:126-139
    if x <= 0.0:
        return a[0] + b[0] * x
    if x >= size:
        h = size / (n - 1)
        slope = b[n - 2] + 2.0 * c[n - 2] * h + 3.0 * d[n - 2] * h * h
        return a[n - 1] + slope * (x - size)
    i = max(min(n - 2, _as_usize((n - 1.0) * x / size)), 0)
    dx = x - size * i / (n - 1)
    return a[i] + b[i] * dx + c[i] * dx * dx + d[i] * dx * dx * dx


def bivariate_interpolate(n_x, n_y, size_x, size_y, mesh, mesh_offset, x, y):    # splines.rs:141-176
    i = max(min(n_x - 2, _as_usize((n_x - 1.0) * x / size_x)), 0)
    dx = x - size_x * i / (n_x - 1)
    dx2 = dx * dx
    grid = MAX_GRID
    raw_mesh_len = n_x * n_y * 2
    block = grid * 4
    offs = 9 + raw_mesh_len + (mesh_offset * n_y * block) + i
    inter = [0.0] * MAX_GRID
    for j in range(n_y):
        rb = offs + j * block
        inter[j] = mesh[rb] + mesh[rb + grid] * dx + mesh[rb + grid * 2] * dx2 + mesh[rb + grid * 3] * dx2 * dx
    a, b, c, d = cubic_spline_coefficients(inter, size_y, n_y)
    return cubic_spline_interpolate(a, b, c, d, n_y, y, size_y)


def interpolate_mesh(x, y, size, mesh):                     # sony.rs:557-563
    n_x, n_y = int(mesh[1]), int(mesh[2])
    return (bivariate_interpolate(n_x, n_y, size[0], size[1], mesh, 0, x, y), bivariate_interpolate(n_x, n_y, size[0], size[1], mesh, 1, x, y))


def _mesh_block(ux, uy, p, mesh):                           # cpu_undistort.rs:169-214: mesh correction, then focal-plane distortion
    fb_inverted = (p.flags & 128) == 128
    fw, fh = F(p.width), F(p.height)
    if len(mesh) > 0 and mesh[0] > 10.0:                    # :169-187
        mesh_size = (mesh[3], mesh[4])
        ox, oy = F(mesh[5]), F(mesh[6])
        cw, ch = F(mesh[7]), F(mesh[8])
        if fb_inverted: uy = fh - uy
        ux = map_coord(ux, 0.0, fw, ox, ox + cw)
        uy = map_coord(uy, 0.0, fh, oy, oy + ch)
        nx, ny = interpolate_mesh(float(ux), float(uy), mesh_size, mesh)
        ux = map_coord(F(nx), ox, ox + cw, 0.0, fw)
        uy = map_coord(F(ny), oy, oy + ch, 0.0, fh)
        if fb_inverted: uy = fh - uy
    # :190-214 FocalPlaneDistortion.  The reference indexes mesh_data[mesh_data[0]] unconditionally (a mesh without the focal-plane block
    # would panic there; sony.rs always appends one); oracle and kernels treat a missing block as "no focal-plane distortion".
    if len(mesh) > 0 and mesh[0] > 0.0 and int(mesh[0]) < len(mesh) and mesh[int(mesh[0])] > 0.0:
        o = int(mesh[0])
        mesh_size = (mesh[3], mesh[4])
        ox, oy = F(mesh[5]), F(mesh[6])
        cw, ch = F(mesh[7]), F(mesh[8])
        stblz_grid = mesh_size[1] / 8.0
        if fb_inverted: uy = fh - uy
        ux = map_coord(ux, 0.0, fw, ox, ox + cw)
        uy = map_coord(uy, 0.0, fh, oy, oy + ch)
        q = float(uy) / stblz_grid
        idx = _as_usize(min(max(math.floor(q), 0.0), 7.0)) if not math.isnan(q) else 0
        delta = float(uy) - stblz_grid * idx
        ux = ux - F(mesh[o + 4 + idx * 2 + 0] * delta)
        uy = uy - F(mesh[o + 4 + idx * 2 + 1] * delta)
        for j in range(idx):
            ux = ux - F(mesh[o + 4 + j * 2 + 0] * stblz_grid)
            uy = uy - F(mesh[o + 4 + j * 2 + 1] * stblz_grid)
        ux = map_coord(ux, ox, ox + cw, 0.0, fw)
        uy = map_coord(uy, oy, oy + ch, 0.0, fh)
        if fb_inverted: uy = fh - uy
    return ux, uy


def rotate_and_distort(px, py, idx, p, m, lens="opencv_fisheye", digital=None, mesh=()):   # cpu_undistort.rs:133-228
    row = m[idx]
    t3 = [F(v) for v in p.translation3d]
    _x = (px * row[0]) + (py * row[1]) + row[2] + t3[0]
    _y = (px * row[3]) + (py * row[4]) + row[5] + t3[1]
    _w = (px * row[6]) + (py * row[7]) + row[8] + t3[2]
    if not (_w > F(0.0)):
        return None
    r_limit_sq = F(p.r_limit) * F(p.r_limit)                 # :521
    if r_limit_sq > 0 and (_x * _x + _y * _y) > r_limit_sq * _w:          # :139 (sic: * _w)
        return None
    lrc = F(p.light_refraction_coefficient)
    if lrc != F(1.0) and lrc > 0:                            # :143-152
        if _w != 0:
            r = sqrtf(_x * _x + _y * _y) / _w
            sin_theta_d = (r / sqrtf(F(1.0) + r * r)) * lrc
            r_d = sin_theta_d / sqrtf(F(1.0) - sin_theta_d * sin_theta_d)
            if r_d != 0:
                _w = _w * (r / r_d)
    k = [F(v) for v in p.k]
    ux, uy = DISTORT[lens](_x, _y, _w, k)
    ux = ux * F(p.f[0]); uy = uy * F(p.f[1])
    if any(row[i] != 0 for i in range(9, 14)):               # IBIS / OIS row :157-165
        ang = row[11]
        cos_a = cosf(-ang); sin_a = sinf(-ang)
        ux, uy = (cos_a * ux - sin_a * uy - row[9] + row[12], sin_a * ux + cos_a * uy - row[10] + row[13])
    ux = ux + F(p.c[0]); uy = uy + F(p.c[1])
    if len(mesh) > 0:
        ux, uy = _mesh_block(ux, uy, p, mesh)
    if digital is not None and (p.flags & 2) == 2:           # :216-220
        ux, uy = DIGITAL[digital](ux, uy, p)
    if F(p.input_horizontal_stretch) > F(0.001): ux = ux / F(p.input_horizontal_stretch)      # :222-223
    if F(p.input_vertical_stretch) > F(0.001): uy = uy / F(p.input_vertical_stretch)
    return ux, uy


def rotate_point(px, py, angle, ox, oy, o2x, o2y):           # cpu_undistort.rs:262-265
    return (cosf(angle) * (px - ox) - sinf(angle) * (py - oy) + o2x, sinf(angle) * (px - ox) + cosf(angle) * (py - oy) + o2y)


def undistort_coord(x, y, p, m, lens="opencv_fisheye", digital=None, mesh=()):   # cpu_undistort.rs:421-517 (incl. the lens-correction blend :429-460)
    ox = map_coord(x, p.output_rect[0], p.output_rect[0] + p.output_rect[2], 0.0, p.output_width)
    oy = map_coord(y, p.output_rect[1], p.output_rect[1] + p.output_rect[3], 0.0, p.output_height)
    ox = ox + F(p.translation2d[0]); oy = oy + F(p.translation2d[1])
    lca = F(p.lens_correction_amount)
    if lca < F(1.0):                                         # :429-460 "add lens distortion back"
        factor = fmaxf(F(1.0) - lca, F(0.001))               # :525-527
        out_cx, out_cy = F(p.output_width) / F(2.0), F(p.output_height) / F(2.0)
        out_fx, out_fy = F(p.f[0]) / F(p.fov) / factor, F(p.f[1]) / F(p.fov) / factor
        nx, ny = ox, oy
        if digital is not None and (p.flags & 2) == 2:       # :432-441 digital warp in the un-zoomed (fov = 1) frame
            fov = F(p.fov)
            uzx, uzy = (nx - out_cx) * fov + out_cx, (ny - out_cy) * fov + out_cy
            d = DIGITAL_UNDISTORT[digital](uzx, uzy, p)
            nx, ny = (d[0] - out_cx) / fov + out_cx, (d[1] - out_cy) / fov + out_cy
        nx, ny = (nx - out_cx) / out_fx, (ny - out_cy) / out_fy
        pt = UNDISTORT[lens](nx, ny, [F(v) for v in p.k])
        if pt is not None:
            nx, ny = pt
        lrc = F(p.light_refraction_coefficient)
        if lrc != F(1.0) and lrc > 0:
            r = sqrtf(nx * nx + ny * ny)
            if r != 0:
                sin_theta_d = (r / sqrtf(F(1.0) + r * r)) / lrc
                r_d = sin_theta_d / sqrtf(F(1.0) - sin_theta_d * sin_theta_d)
                fac = r_d / r
                nx, ny = nx * fac, ny * fac
        nx, ny = nx * out_fx + out_cx, ny * out_fy + out_cy
        ox, oy = nx * (F(1.0) - lca) + ox * lca, ny * (F(1.0) - lca) + oy * lca
    hrs = (p.flags & 16) == 16
    sy = max(min(as_i32(round_half_away(ox)), p.width), 0) if hrs else max(min(as_i32(round_half_away(oy)), p.height), 0)
    if p.matrix_count > 1:
        pt = rotate_and_distort(ox, oy, p.matrix_count // 2, p, m, lens, digital, mesh)
        if pt is not None:
            sy = max(min(as_i32(round_half_away(pt[0])), p.width), 0) if hrs else max(min(as_i32(round_half_away(pt[1])), p.height), 0)
    idx = min(sy, p.matrix_count - 1)
    uv = rotate_and_distort(ox, oy, idx, p, m, lens, digital, mesh)
    if uv is None:
        return None
    u, v = uv
    fw, fh = F(p.width), F(p.height)
    if F(p.input_rotation) != 0:                             # :485-491
        rotation = F(p.input_rotation) * (F(math.pi) / F(180.0))
        sw, sh = fw, fh
        fw, fh = rotate_point(sw, sh, rotation, F(0.0), F(0.0), F(0.0), F(0.0))
        fw, fh = round_half_away(abs(fw)), round_half_away(abs(fh))
        u, v = rotate_point(u, v, rotation, sw / F(2.0), sh / F(2.0), fw / F(2.0), fh / F(2.0))
    width_f, height_f = F(p.width), F(p.height)
    if p.background_mode == 1:                               # edge repeat :495-499
        u = min(max(u, F(3.0)), width_f - F(3.0)); v = min(max(v, F(3.0)), height_f - F(3.0))
    elif p.background_mode == 2:                             # edge mirror :500-509
        rx, ry = round_half_away(u), round_half_away(v)
        width3, height3 = width_f - F(3.0), height_f - F(3.0)
        if rx > width3: u = width3 - (rx - width3)
        if rx < F(3.0): u = F(3.0) + width_f - (width3 + rx)
        if ry > height3: v = height3 - (ry - height3)
        if ry < F(3.0): v = F(3.0) + height_f - (height3 + ry)
    if p.background_mode != 3:                               # :510-515
        u = map_coord(u, 0.0, fw, p.source_rect[0], p.source_rect[0] + p.source_rect[2])
        v = map_coord(v, 0.0, fh, p.source_rect[1], p.source_rect[1] + p.source_rect[3])
    return u, v


def sample_bilinear(u, v, src, p, bg, count, sbytes=1):   # cpu_undistort.rs:370-418 with I = 2; src: flat array of scalars
    sx0 = as_i32(round_half_away(u * F(32.0))); sy0 = as_i32(round_half_away(v * F(32.0)))
    sx, sy = sx0 >> 5, sy0 >> 5
    fx, fy = sx0 & 31, sy0 & 31
    cx = [F(1.0) - F(fx) / F(32.0), F(fx) / F(32.0)]         # COEFFS[frac * 2 ..] (cpu_undistort.rs:14-19)
    cy = [F(1.0) - F(fy) / F(32.0), F(fy) / F(32.0)]
    rx0, ry0 = p.source_rect[0], p.source_rect[1]
    rx1, ry1 = rx0 + p.source_rect[2], ry0 + p.source_rect[3]
    total = [F(0.0)] * 4
    for yp in range(2):
        if ry0 <= sy + yp < ry1:
            xsum = [F(0.0)] * 4
            for xp in range(2):
                if rx0 <= sx + xp < rx1:
                    off = ((sy + yp) * p.stride + (sx + xp) * p.bytes_per_pixel) // sbytes          # index in scalars
                    px = [F(src[off + c]) if c < count else F(0.0) for c in range(4)]
                else:
                    px = bg
                xsum = [xsum[c] + px[c] * cx[xp] for c in range(4)]
            total = [total[c] + xsum[c] * cy[yp] for c in range(4)]
        else:
            total = [total[c] + bg[c] * cy[yp] for c in range(4)]
    lim = F(p.pixel_value_limit)
    return [min(t, lim) if not math.isnan(float(t)) else lim for t in total]


_COEFF_TABLES = {}


def _coeffs(I):
    """COEFFS of cpu_undistort.rs:21-58 (bicubic: 32 x 4, Lanczos4: 32 x 8) — the literals, parsed from the generated table the build
    checks against the reference's 448 values (oracle/gen_coeffs.py --check-reference)."""
    if not _COEFF_TABLES:
        import os, re
        txt = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "gf_coeffs.inc")).read()
        for name, key in (("GF_COEFFS_BICUBIC", 4), ("GF_COEFFS_LANCZOS4", 8)):
            body = txt[txt.index(name):]
            body = body[body.index("{") + 1:body.index("}")]
            _COEFF_TABLES[key] = [F(v) for v in re.findall(r"-?\d+\.\d+", body)]
    return _COEFF_TABLES[I]


def sample_separable(u, v, src, p, bg, count, sbytes, I):   # cpu_undistort.rs:370-418 with I = 4 (bicubic) or 8 (Lanczos4)
    offset = F(1.0) if I == 4 else F(3.0)
    tab = _coeffs(I)
    u = u - offset; v = v - offset
    sx0 = as_i32(round_half_away(u * F(32.0))); sy0 = as_i32(round_half_away(v * F(32.0)))
    sx, sy = sx0 >> 5, sy0 >> 5
    cx = tab[(sx0 & 31) * I:(sx0 & 31) * I + I]; cy = tab[(sy0 & 31) * I:(sy0 & 31) * I + I]
    rx0, ry0 = p.source_rect[0], p.source_rect[1]
    rx1, ry1 = rx0 + p.source_rect[2], ry0 + p.source_rect[3]
    total = [F(0.0)] * 4
    for yp in range(I):
        if ry0 <= sy + yp < ry1:
            xsum = [F(0.0)] * 4
            for xp in range(I):
                if rx0 <= sx + xp < rx1:
                    off = ((sy + yp) * p.stride + (sx + xp) * p.bytes_per_pixel) // sbytes
                    px = [F(src[off + c]) if c < count else F(0.0) for c in range(4)]
                else:
                    px = bg
                xsum = [xsum[c] + px[c] * cx[xp] for c in range(4)]
            total = [total[c] + xsum[c] * cy[yp] for c in range(4)]
        else:
            total = [total[c] + bg[c] * cy[yp] for c in range(4)]
    lim = F(p.pixel_value_limit)
    return [min(t, lim) if not math.isnan(float(t)) else lim for t in total]


# ---- EWA (elliptical weighted average) CubicBC resampler: cpu_undistort.rs:271-369 ----
def affine_bbox(jac):                        # :274-279
    jx, jy, jz, jw = jac
    return (F(2.0) * fmaxf(fmaxf(abs(jx + jy), abs(jx - jy)), F(1.0)), F(2.0) * fmaxf(fmaxf(abs(jz + jw), abs(jz - jw)), F(1.0)))


def clamped_ellipse(jac):                    # :281-314
    jx, jy, jz, jw = jac
    f0 = abs(jx * jw - jy * jz)
    f = fmaxf(f0 * f0, F(0.1))
    a = (jz * jz + jw * jw) / f
    b = F(-2.0) * (jx * jz + jy * jw) / f
    c = (jx * jx + jy * jy) / f
    vx, vy = c - a, -b
    lv = sqrtf(vx * vx + vy * vy)
    v0 = vx / lv if lv > F(0.01) else F(1.0)
    cc = sqrtf(fmaxf(F(1.0) + v0, F(0.0)) / F(2.0))
    s = sqrtf(fmaxf(F(1.0) - v0, F(0.0)) / F(2.0))
    a0 = a * cc * cc - b * cc * s + c * s * s
    c0 = a * s * s + b * cc * s + c * cc * cc
    bt1 = b * (cc * cc - s * s)
    bt2 = F(2.0) * (a - c) * cc * s
    b0 = bt1 + bt2
    b0v2 = bt1 - bt2
    if abs(b0) > abs(b0v2):
        s = -s
        b0 = b0v2
    a0 = fminf(a0, F(1.0))
    c0 = fminf(c0, F(1.0))
    sn = -s
    return (a0 * cc * cc - b0 * cc * sn + c0 * sn * sn,
            F(2.0) * a0 * cc * sn + b0 * cc * cc - b0 * sn * sn - F(2.0) * c0 * cc * sn,
            a0 * sn * sn + b0 * cc * sn + c0 * cc * cc)


def bc2(x, p):                               # :316-326
    x = abs(x)
    x2 = x * x
    cp = [F(v) for v in p.ewa_coeffs_p]; cq = [F(v) for v in p.ewa_coeffs_q]
    if x < F(1.0):
        return cp[0] + cp[1] * x + cp[2] * x2 + cp[3] * x2 * x
    elif x < F(2.0):
        return cq[0] + cq[1] * x + cq[2] * x2 + cq[3] * x2 * x
    return F(0.0)


def sample_ewa(u, v, jac, src, p, bg, count, sbytes):       # :331-369
    tx, ty = affine_bbox(jac)
    b0 = as_i32(F(math.floor(float(u - tx)))); b1 = as_i32(F(math.ceil(float(u + tx))))
    b2 = as_i32(F(math.floor(float(v - ty)))); b3 = as_i32(F(math.ceil(float(v + ty))))
    total = [F(0.0)] * 4
    sum_div = F(0.0)
    A, B, C = clamped_ellipse(jac)
    rx0, ry0 = p.source_rect[0], p.source_rect[1]
    rx1, ry1 = rx0 + p.source_rect[2], ry0 + p.source_rect[3]
    for in_y in range(b2, b3 + 1):
        in_fy = F(in_y) - v
        in_fy2 = in_fy * B
        in_fy3 = in_fy * in_fy * C
        for in_x in range(b0, b1 + 1):
            in_fx = F(in_x) - u
            dr = in_fx * in_fx * A + in_fx * in_fy2 + in_fy3
            k = bc2(sqrtf(dr), p)
            if k == 0:
                continue
            if ry0 <= in_y < ry1 and rx0 <= in_x < rx1:
                off = (in_y * p.stride + in_x * p.bytes_per_pixel) // sbytes
                px = [F(src[off + c]) if c < count else F(0.0) for c in range(4)]
            else:
                px = bg
            total = [total[c] + k * px[c] for c in range(4)]
            sum_div = sum_div + k
    total = [t / sum_div for t in total]
    lim = F(p.pixel_value_limit)             # :413-418 applies to every resampler
    return [fminf(t, lim) for t in total]


def remap_colorrange(px, is_y):              # :254-260
    s = F(0.85882352) if is_y else F(0.87843137)
    px = [v * s for v in px]
    px[0] = px[0] + F(16.0)
    px[1] = px[1] + F(16.0)
    return px


def to_u8(v):                                # `as u8`: truncate, saturate, NaN -> 0
    v = float(v)
    if math.isnan(v):
        return 0
    return max(0, min(255, int(v)))


def to_scalar(v, sdt):                       # PixelType::from_float: Rust `as u8` / `as u16` (truncate, saturate, NaN -> 0); f32 passes through
    if sdt == np.float32:
        return F(v)
    v = float(v)
    if math.isnan(v):
        return 0
    return max(0, min(255 if sdt == np.uint8 else 65535, int(v)))


def _sample(u, v, jac, flat, p, bg, count, sbytes):
    if p.interpolation > 8:
        return sample_ewa(u, v, jac, flat, p, bg, count, sbytes)
    if p.interpolation == 2:
        return sample_bilinear(u, v, flat, p, bg, count, sbytes)
    return sample_separable(u, v, flat, p, bg, count, sbytes, p.interpolation)


def undistort_image(src, dst, p, matrices, lens="opencv_fisheye", sdt=np.uint8, digital=None, mesh=None):
    """src, dst: 2-D uint8 arrays (rows x stride).  Writes dst in place like the reference (only pixels it touches) — the main loop
    cpu_undistort.rs:543-625.  sdt: the scalar type of a channel (np.uint8, np.uint16 or np.float32); mesh: the f32 mesh or None."""
    m = [[F(x) for x in row] for row in np.asarray(matrices, dtype=np.float32).reshape(-1, 14)]
    mesh64 = [float(v) for v in np.asarray(mesh, dtype=np.float32)] if mesh is not None else []       # :539 widened once
    sbytes = np.dtype(sdt).itemsize
    count = p.bytes_per_pixel // sbytes
    flat = src.reshape(-1).view(sdt)
    dview = dst.view(sdt)                    # rows x (stride / sbytes) scalars (strides are multiples of the scalar size in these tests)
    bg = [F(p.background[c]) * F(p.max_pixel_value) for c in range(4)]
    fill_bg = (p.flags & 4) == 4
    fix_range = (p.flags & 1) == 1
    is_y = p.plane_index == 0
    for y in range(dst.shape[0]):
        npix = min(dst.shape[1], p.output_stride) // p.bytes_per_pixel
        for x in range(npix):
            opx = map_coord(x, p.output_rect[0], p.output_rect[0] + p.output_rect[2], 0.0, p.output_width)
            opy = map_coord(y, p.output_rect[1], p.output_rect[1] + p.output_rect[3], 0.0, p.output_height)
            if not (opx >= 0 and opy >= 0 and as_i32(opx) < p.output_width and as_i32(opy) < p.output_height):
                continue
            if fill_bg:                                                                   # :559-562
                for c in range(count):
                    dview[y, x * count + c] = to_scalar(bg[c], sdt)
                continue
            pixel = bg
            uv = undistort_coord(F(x), F(y), p, m, lens, digital, mesh64)
            if uv is not None:
                jac = (F(1.0), F(0.0), F(0.0), F(1.0))
                if p.interpolation > 8:                                                   # :567-572 forward differences, None -> (0, 0)
                    eps = F(0.01)
                    a = undistort_coord(F(x) + eps, F(y), p, m, lens, digital, mesh64) or (F(0.0), F(0.0))
                    b = undistort_coord(F(x), F(y) + eps, p, m, lens, digital, mesh64) or (F(0.0), F(0.0))
                    xyx = (a[0] - uv[0], a[1] - uv[1]); xyy = (b[0] - uv[0], b[1] - uv[1])
                    jac = (xyx[0] / eps, xyy[0] / eps, xyx[1] / eps, xyy[1] / eps)
                u, v = uv
                if p.background_mode == 3:                                                # :576-611 margin with feather
                    width_f, height_f = F(p.width), F(p.height)
                    widthf, heightf = width_f - F(1.0), height_f - F(1.0)
                    feather = fmaxf(F(p.background_margin_feather) * heightf, F(0.0001))
                    p2x, p2y = u, v
                    alpha = F(1.0)
                    if (u > widthf - feather) or (u < feather) or (v > heightf - feather) or (v < feather):
                        alpha = fmaxf(fminf(fminf(fminf(fminf(widthf - u, heightf - v), u), v) / feather, F(1.0)), F(0.0))
                        p2x, p2y = p2x / width_f, p2y / height_f
                        mg = F(1.0) - F(p.background_margin)
                        p2x, p2y = ((p2x - F(0.5)) * mg) + F(0.5), ((p2y - F(0.5)) * mg) + F(0.5)
                        p2x, p2y = p2x * width_f, p2y * height_f
                    fw, fh = width_f, height_f
                    if F(p.input_rotation) != 0:
                        rotation = F(p.input_rotation) * (F(math.pi) / F(180.0))
                        fw, fh = rotate_point(fw, fh, rotation, F(0.0), F(0.0), F(0.0), F(0.0))
                        fw, fh = round_half_away(abs(fw)), round_half_away(abs(fh))
                    sr = p.source_rect
                    u, v = map_coord(u, 0.0, fw, sr[0], sr[0] + sr[2]), map_coord(v, 0.0, fh, sr[1], sr[1] + sr[3])
                    p2x, p2y = map_coord(p2x, 0.0, fw, sr[0], sr[0] + sr[2]), map_coord(p2y, 0.0, fh, sr[1], sr[1] + sr[3])
                    c1 = _sample(u, v, jac, flat, p, bg, count, sbytes)
                    c2 = _sample(p2x, p2y, jac, flat, p, bg, count, sbytes)
                    pixel = [c1[c] * alpha + c2[c] * (F(1.0) - alpha) for c in range(4)]
                else:
                    pixel = _sample(u, v, jac, flat, p, bg, count, sbytes)
            if fix_range:
                pixel = remap_colorrange(list(pixel), is_y)
            for c in range(count):
                dview[y, x * count + c] = to_scalar(pixel[c], sdt)
