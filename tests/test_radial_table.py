"""The filtered pre-pass's per-lens radial table (build_radial_table in filter_prepass.cu, read by Lens2<opencv_fisheye>::approx_v), replayed on the
host through gf_filter_radial_table: which rows are fitted, which repeat the first fitted row and which are NaN, the rounded r^2 cap, and
the fit error against R(a) = T(a) s(theta) off the 65 points per row the host checks."""
import ctypes as C
import math

import numpy as np
import pytest

import gyroflow_b200 as g

ROWS, FIT, FIT_ROWS = 8192, (127 - 30) << 4, 44 * 16
BUDGET = 2.0 ** -23             # the host's budget on the table error (profiles/FILTER_ANALYSIS.md step 3)


def table(k):
    lib = g.load_library()
    kk = (C.c_float * 4)(*k)
    rows = np.zeros((ROWS, 4), np.float32)
    cap = C.c_float()
    assert lib.gf_filter_radial_table(kk, rows.ctypes.data_as(C.c_void_p), ROWS, C.byref(cap)) == ROWS
    return rows, cap.value


def conditioning_cap(k):
    """filter_a_cap restated: tan^2 of the largest angle <= 1.55 at which sum |k_i| t^(2i+2) <= 1/4, or 0 below 0.5 rad"""
    B = lambda t: sum(abs(float(k[i])) * t ** (2 * i + 2) for i in range(4))
    lo, hi = 0.0, 1.55
    if B(hi) > 0.25:
        for _ in range(60):
            mid = 0.5 * (lo + hi)
            lo, hi = (mid, hi) if B(mid) <= 0.25 else (lo, mid)
    else:
        lo = hi
    return 0.0 if lo < 0.5 else float(np.float32(min(math.tan(lo) ** 2 * 0.999, 16000.0)))


def R(a, k):
    r = math.sqrt(a)
    T = 1.0 - a / 3.0 + a * a / 5.0 if r < 1e-4 else math.atan(r) / r
    q = a * T * T
    return T * (1.0 + q * (k[0] + q * (k[1] + q * (k[2] + q * k[3]))))


def lenses():
    rng = np.random.default_rng(11)
    out = [[0.0, 0.0, 0.0, 0.0], [0.02, -0.01, 0.004, -0.001], [-0.25, 0.0, 0.0, 0.0]]
    for j in range(4):                                   # one-term lenses at the smallest cap the filter accepts (0.5 rad)
        for sgn in (1.0, -1.0):
            k = [0.0] * 4
            k[j] = sgn * 0.25 / 0.5 ** (2 * j + 2) * 0.999
            out.append(k)
    for _ in range(12):                                  # random signs, scaled to reach the conditioning cap between 0.5 and 1.55 rad
        k = (rng.random(4) * 2 - 1) * 0.35 ** np.arange(4)
        t2 = (0.5 + 1.05 * rng.random()) ** 2
        k = k * 0.25 / (t2 * (abs(k[0]) + t2 * (abs(k[1]) + t2 * (abs(k[2]) + t2 * abs(k[3])))))
        out.append([float(np.float32(v)) for v in k])
    return out


@pytest.mark.parametrize("k", lenses())
def test_rows_and_cap(k):
    rows, cap = table(k)
    want = conditioning_cap(np.float32(k))
    assert want > 0.0 and cap > 0.0, "every lens inside the conditioning cap meets the error budget"
    cap_bits = int(np.float32(cap).view(np.uint32))
    assert cap_bits & 0x7ffff == 0 and cap <= want and int(np.float32(want).view(np.uint32)) >> 19 == cap_bits >> 19
    n_valid = (cap_bits >> 19) - FIT
    assert 0 < n_valid <= FIT_ROWS
    assert np.isfinite(rows[FIT:FIT + n_valid]).all()
    assert np.isnan(rows[FIT + n_valid:]).all()                      # r^2 >= cap, beyond 2^14, NaN and the sign bit: never certified
    assert (rows[:FIT] == rows[FIT]).all()                            # below 2^-30: the first fitted row


@pytest.mark.parametrize("k", lenses())
def test_fit_error_off_the_checked_points(k):
    """The f32 coefficients' cubic in d = a - lo, evaluated in f64, against R at points between the host's 65 per row"""
    rows, cap = table(k)
    n_valid = (int(np.float32(cap).view(np.uint32)) >> 19) - FIT
    rng = np.random.default_rng(5)
    worst = 0.0
    for i in range(0, n_valid, 3):
        e, j = divmod(i, 16)
        lo = math.ldexp(1.0 + j / 16.0, e - 30)
        hi = math.ldexp(1.0 + (j + 1) / 16.0, e - 30)
        c = [float(v) for v in rows[FIT + i]]
        for a in np.float32(lo + (hi - lo) * rng.random(16)):
            a = float(a)
            d = a - lo
            v = c[0] + d * (c[1] + d * (c[2] + d * c[3]))
            worst = max(worst, abs(v / R(a, k) - 1.0))
    assert worst <= BUDGET, worst


def test_row_of_every_bit_pattern():
    """approx_v indexes the table with bits(a) >> 19 unclamped: an 8192-row table covers every pattern, and the row of a NaN or of any
    a at or above the cap is NaN, so the certificate fails there"""
    rows, cap = table([0.05, -0.02, 0.003, 0.0])
    for a in (np.float32(cap), np.float32(2.0 ** 14), np.float32(np.inf), np.float32(np.nan), np.float32(-np.nan), np.float32(-1.0)):
        assert np.isnan(rows[int(a.view(np.uint32)) >> 19]).all()
    for a in (np.float32(0.0), np.float32(1e-45), np.float32(2.0 ** -31), np.float32(0.25)):
        assert np.isfinite(rows[int(a.view(np.uint32)) >> 19]).all()


def test_strongly_curved_lens_has_no_table():
    """A lens too strongly curved for the filter (conditioning cap below 0.5 rad) runs without it"""
    rows, cap = table([40.0, 0.0, 0.0, 0.0])
    assert cap == 0.0 and np.isnan(rows).all()
