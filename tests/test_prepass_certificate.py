"""The certify-and-round step of the filtered rolling-shutter pre-pass (certify_row in warp_kernel_x2.cuh).

The packed kernel evaluates the mid-row v of a pixel approximately (t, with a proven error bound eps) and keeps the pair on the fast
path only when every real t' within eps of t selects the same matrix row, max(min(round_half_away(t'), lim), 0).  certify_row decides
that and yields the row from one rounding: s = RN(t + 1.5 * 2^23), r = t - (s - 1.5 * 2^23), certified iff RD(1/2 - |r|) > eps and
|t| < 2^20, row = clamp(bits(s) - bits(1.5 * 2^23), 0, lim).

CPU part: an exact numpy emulation of that predicate is checked against the rounding it stands for over EVERY float with |t| < 2^20.
GPU part: the device function itself, on the same inputs, must equal the emulation bit for bit.
"""
import ctypes as C

import numpy as np
import pytest

M = np.float32(12582912.0)                       # 1.5 * 2^23
M_BITS = 0x4B400000
# eps of the kernel: rho |t - c_y| + 2^-22 |t| with rho = 2^-17 and |t| < 2^20.  With c_y inside a frame of up to 2^16 rows this is
# below (2^20 + 2^16) 2^-17 + 2^20 2^-22 = 8.75; the float just above covers the rounding of the fused multiply-add.
EPS_MAX = float(np.nextafter(np.float32(8.75), np.float32(np.inf)))
EPS = [0.0, 2.0 ** -30, 0.0087, EPS_MAX]
LIM = 1 << 16                                    # the row clamp of a frame of 2^16 rows
T_LIMIT_BITS = 0x49800000                        # bits of 2^20


def _sub_rd_half(a):
    """RD(0.5 - a) in float32 for float32 a >= 0 (the device's __fsub_rd(0.5f, |r|))."""
    d = np.float32(0.5) - a                                             # round to nearest
    above = d.astype(np.float64) + a.astype(np.float64) > 0.5          # RN went above the exact value (sum exact for a >= 2^-26)
    d = np.where(above, np.nextafter(d, np.float32(-np.inf)), d)
    tiny = (a > 0) & (a < np.float32(2.0 ** -26))                        # 0.5 - a in (0.5 - 2^-26, 0.5): RD is the float below 1/2
    return np.where(tiny, np.float32(0.5 - 2.0 ** -25), d).astype(np.float32)


def certify_row_np(t, eps, lim):
    """Emulation of certify_row: (certified, row) for float32 array t."""
    with np.errstate(invalid="ignore", over="ignore"):
        s = t + M
        r = t - (s - M)
        d = _sub_rd_half(np.abs(r))
        cert = (d > np.float32(eps)) & (np.abs(t) < np.float32(2.0 ** 20))
        row = np.maximum(np.minimum(s.view(np.int32).astype(np.int64) - M_BITS, lim), 0)
    return cert, row


def _truth(t, lim):
    """For float32 t: the clamped half-away row, and the distances from t to the nearest row boundaries below (>= 0) and above (> 0)
    at which that clamped row changes (inf where there is none).  Boundaries are j - 1/2, j = 1..lim (t' = j - 1/2 has row j)."""
    t64 = t.astype(np.float64)
    k = np.floor(t64 + 0.5)                      # j - 1/2 <= t < j + 1/2  <=>  j = k
    row = np.clip(k, 0, lim).astype(np.int64)    # negative t: round half away gives <= 0, clamped to 0 like k
    j_lo = np.minimum(k, lim)
    dist_lo = np.where(j_lo >= 1, t64 - (j_lo - 0.5), np.inf)
    j_hi = np.maximum(k + 1, 1)
    dist_hi = np.where(j_hi <= lim, (j_hi - 0.5) - t64, np.inf)
    return row, dist_lo, dist_hi


def test_certify_row_exhaustive():
    """Every float t with |t| < 2^20, each eps: a certified t yields round_half_away(t) clamped, and no real t' within eps of t yields
    another clamped row.  Also: the certificate is not vacuous (it accepts all but a sliver for small eps)."""
    chunk = 1 << 23
    certified = {e: 0 for e in EPS}
    total = 0
    for sign in (0, 0x80000000):
        for lo in range(0, T_LIMIT_BITS, chunk):
            bits = np.arange(lo, min(lo + chunk, T_LIMIT_BITS), dtype=np.uint32) | np.uint32(sign)
            t = bits.view(np.float32)
            total += t.size
            with np.errstate(invalid="ignore", over="ignore"):
                s = t + M
                r = t - (s - M)
                d = _sub_rd_half(np.abs(r))
                row = np.maximum(np.minimum(s.view(np.int32).astype(np.int64) - M_BITS, LIM), 0)
            want_row, dist_lo, dist_hi = _truth(t, LIM)
            for e in EPS:
                cert = d > np.float32(e)
                certified[e] += int(np.count_nonzero(cert))
                safe = (dist_lo >= e) & (dist_hi > e) & (row == want_row)
                bad = cert & ~safe
                if bad.any():
                    i = int(np.flatnonzero(bad)[0])
                    pytest.fail("eps %r: t = %r certified with row %d, want %d, boundary distances %r / %r"
                                % (e, float(t[i]), int(row[i]), int(want_row[i]), float(dist_lo[i]), float(dist_hi[i])))
    assert total == 2 * T_LIMIT_BITS
    assert certified[0.0] > total - (1 << 22)                   # only the ties n + 1/2 (|n| < 2^20 and exact in float) are refused
    assert certified[0.0087] > 0.9 * total                      # most floats are tiny, far from every boundary


def _sample_inputs(rng):
    """A few million float32 inputs: random bit patterns with |t| < 2^20, neighbours of half-integers and of the eps-boundaries of the
    tested eps, tiny and subnormal values, signed zeros, and values outside the certificate's domain (large, inf, NaN)."""
    parts = [rng.integers(0, T_LIMIT_BITS, 1 << 21, dtype=np.uint32) | (rng.integers(0, 2, 1 << 21, dtype=np.uint32) << 31)]
    n = rng.integers(-70000, 70000, 1 << 18).astype(np.float64)
    for off in [0.5, -0.5] + [0.5 + e for e in EPS] + [0.5 - e for e in EPS]:
        c = (n + off).astype(np.float32)
        steps = rng.integers(-3, 4, c.size).astype(np.int32)
        parts.append((c.view(np.int32) + steps).view(np.uint32))
    parts.append(rng.integers(0, 0x33000000, 1 << 18, dtype=np.uint32))                    # |t| < 2^-25, subnormals included
    parts.append(rng.integers(0x49800000, 0x80000000, 1 << 16, dtype=np.uint32))           # |t| >= 2^20, inf, NaN
    parts.append(np.array([0, 0x80000000, 0x3F000000, 0xBF000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x497FFFFF, 0x49800000], np.uint32))
    return np.concatenate(parts).view(np.float32)


@pytest.mark.gpu
def test_certify_row_device_matches_emulation():
    """gf_cuda_selftest_certify runs certify_row — the function the packed kernel calls — on the device; certificate and row must equal
    the emulation above for every input (rows compared for finite t: the device's NaN bits are not the host's)."""
    import gyroflow_b200 as g
    lib = g.load_library()
    t = np.ascontiguousarray(_sample_inputs(np.random.default_rng(20261016)))
    finite = np.isfinite(t)
    for eps in EPS:
        for lim in (LIM, 2159, 0):
            cert = np.zeros(t.size, np.uint8)
            row = np.zeros(t.size, np.int32)
            assert lib.gf_cuda_selftest_certify(0, t.ctypes.data_as(C.c_void_p), t.size, C.c_float(eps), lim,
                                                cert.ctypes.data_as(C.c_void_p), row.ctypes.data_as(C.c_void_p)) == 0
            want_cert, want_row = certify_row_np(t, eps, lim)
            assert np.array_equal(cert.astype(bool), want_cert), (eps, lim, t[cert.astype(bool) != want_cert][:8])
            assert np.array_equal(row[finite], want_row[finite]), (eps, lim, t[finite][row[finite] != want_row[finite]][:8])
