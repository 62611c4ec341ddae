"""Second transcription of OptimSync (src/core/synchronization/optimsync.rs), in numpy — TESTS ONLY.

The exact stages (resampling, blackman with glibc cosf, rank, masks, NMS, segments) are written independently of the C oracle
(oracle/gf_oracle_optsync.c) so the two can be compared bit for bit.  The spectral stage has no exact oracle: bands_f64 takes the DFT in
f64 (scipy.fft) of the exact f32 windowed inputs, and `bar` bounds how far an f32 FFT's band energies can be from it (DESIGN.md §7).
`margins` reports how far each decision of the selection is from flipping under that bar.
"""
import ctypes as C
import ctypes.util
import math

import numpy as np
import scipy.fft

STEP = 16
F32 = np.float32
U = 2.0 ** -24                           # f32 unit roundoff

_libm = C.CDLL(ctypes.util.find_library("m"))
_libm.cosf.restype = C.c_float
_libm.cosf.argtypes = [C.c_float]


def as_usize(x):
    """`x as usize` for f64: saturating, NaN 0."""
    if x != x or x <= 0.0:
        return 0
    return min(int(x), 2 ** 64 - 1)


def resample(ts, gyro, has_gyro=None):
    """OptimSync::new (:30-66): (avg_sr, n_res x 3 float64)."""
    ts = np.asarray(ts, np.float64); gyro = np.asarray(gyro, np.float64).reshape(-1, 3)
    has = np.ones(ts.size, bool) if has_gyro is None else np.asarray(has_gyro).astype(bool)
    duration = ts[-1] - ts[0]
    avg_sr = float(np.count_nonzero(has)) / duration * 1000.0
    n_res = as_usize(duration * avg_sr / 1000.0)
    g = np.where(has[:, None], gyro, 0.0)                                  # unwrap_or_default
    t = np.arange(n_res, dtype=np.float64) * 1000.0 / avg_sr
    i_r = np.minimum(np.searchsorted(ts, t, side="left"), ts.size - 1)     # partition_point(|s| s.ts < t).min(len - 1)
    i_l = np.maximum(i_r, 1) - 1
    tl, tr = ts[i_l][:, None], ts[i_r][:, None]
    with np.errstate(all="ignore"):
        interp = (g[i_l] * (tr - t[:, None]) + g[i_r] * (t[:, None] - tl)) / (tr - tl)
    out = np.where((i_l == i_r)[:, None], g[i_l], interp)
    return avg_sr, out


def blackman(width):
    """blackman (:15-27) in f32; f32::cos is glibc cosf, which numpy's float32 cos is not."""
    a0, a1, a2 = F32(7938.0) / F32(18608.0), F32(9240.0) / F32(18608.0), F32(1430.0) / F32(18608.0)
    pi = F32(math.pi)
    size = F32(width - 1)
    n = np.arange(width).astype(F32)
    x1 = F32(2.0) * pi * n / size
    x2 = F32(4.0) * pi * n / size
    c1 = np.array([_libm.cosf(float(v)) for v in x1], F32)
    c2 = np.array([_libm.cosf(float(v)) for v in x2], F32)
    return a0 - a1 * c1 + a2 * c2


def map_to_bin(N, sr, f):
    v = round_half_away(N / sr * f)
    return int(min(max(v, 0.0), float(N // 2 - 1)))


def round_half_away(x):
    return math.copysign(math.floor(abs(x) + 0.5), x) if abs(x) < 2 ** 52 else x


def nlfunc(arg, trip):
    with np.errstate(invalid="ignore"):
        return np.where(arg < trip, F32(0.0), arg - trip).astype(F32)


def ranks(bands):
    """rank (:141-155) in f32: (rank, low_motion)."""
    b = np.asarray(bands, F32).reshape(-1, 3)
    lf, mf, hf = b[:, 0], b[:, 1], b[:, 2]
    mf_max = F32(np.fmax.reduce(mf, initial=F32(0.0))) if mf.size else F32(0.0)
    low = bool(mf_max < F32(50.0))
    k = F32(0.003); one = F32(1.0)
    with np.errstate(all="ignore"):
        if low:
            r = (lf + mf) / (one + nlfunc(hf, F32(450.0)) * k)
        else:
            r = mf / (one + nlfunc(hf, F32(450.0)) * k) / (one + nlfunc(lf, F32(650.0)) * k)
    return r.astype(F32), low


def masked(rank, sr, trim):
    """The masks (:158-176): rank < 50, outside every trim range, the first / last 2 s of a log over 12 s."""
    ratio = STEP / sr
    n = rank.size
    time = np.arange(n, dtype=np.float64) * ratio
    inside = np.zeros(n, bool)
    for a, b in np.asarray(trim, np.float64).reshape(-1, 2):
        inside |= (time >= a) & (time <= b)
    r = rank.copy()
    with np.errstate(invalid="ignore"):
        r[(r < F32(50.0)) | ~inside] = F32(0.0)
    total = n * ratio
    if total > 12.0:
        r[(time < 2.0) | (time >= total - 2.0)] = F32(0.0)
    return r, ratio


def nms(rank, radius):
    """The NMS double loop (:178-185) by offset d = i - j: j in [max(0, i - r), min(i + r, len - 1)) means -r < d <= r, j < len - 1."""
    n = rank.size
    sup = np.zeros(n, bool)
    for d in range(-radius + 1, radius + 1):
        j = np.arange(max(0, -d), min(n - 1, n - d))
        if j.size:
            with np.errstate(invalid="ignore"):
                sup[j] |= rank[j] < rank[j + d]
    out = rank.copy()
    out[sup] = F32(0.0)
    return out


def select(bands, sr, N, target, trim):
    """run after the spectra: (points_ms, rank_clone, ratio)."""
    rank, _ = ranks(bands)
    r, ratio = masked(rank, sr, trim)
    rn = nms(r, as_usize(sr / 16.0 / 2.0 * 8.0))
    n = rn.size
    seg = (n + target - 1) // target
    pts = []
    for s in range(target):
        start = s * seg; end = min(start + seg, n)
        if start >= end:
            continue
        best = start
        for j in range(start + 1, end):
            if not (rn[best] > rn[j]):          # max_by(partial_cmp, NaN -> Equal): the last of equal elements
                best = j
        if rn[best] < F32(0.1):
            continue
        pts.append((best * 16.0 + N / 2.0) / sr * 1000.0)
    return np.array(pts, np.float64), rank, ratio


def sizes(ts, has_gyro=None):
    sr, g = resample(ts, np.zeros((len(ts), 3)), has_gyro)
    N = int(round_half_away(sr))
    nr = g.shape[0]
    return sr, N, nr, (nr - N) // STEP + 1 if nr >= N else 0


# ---- spectra and the bar ----

def scale_f32(N):
    return float(F32(np.sqrt(F32(1.0) / F32(N))) / F32(N) * F32(256.0))


def _windows(g32, N, idx):
    win = blackman(N)
    starts = np.asarray(idx, np.int64) * STEP
    seg = np.stack([g32[s:s + N] for s in starts]) if len(starts) else np.zeros((0, N, 3), F32)   # w x N x 3
    return (seg * win[None, :, None]).astype(F32)


def _half_pairs(X, N):
    h = N // 2
    k = np.arange(h)
    return X[..., k] + X[..., N - 1 - k]           # zip(iter, iter.rev()).take(N / 2)


def bands_f64(g32, N, sr, idx):
    """Per window in idx: f64 band energies (w x 3) of the exact f32 windowed inputs, the ℓ2 norm of each axis's spectrum (w x 3) and the
    number of bins of each band."""
    xw = _windows(g32, N, idx).astype(np.float64).transpose(0, 2, 1)       # w x 3 x N
    X = scipy.fft.fft(xw, axis=-1)
    mag = np.abs(_half_pairs(X, N)) * scale_f32(N)                          # w x 3 x N/2
    b = [0, map_to_bin(N, sr, 2.0), map_to_bin(N, sr, 30.0), map_to_bin(N, sr, 2000.0)]
    merged = mag.sum(axis=1)
    out = np.stack([merged[:, b[i]:b[i + 1]].sum(axis=1) for i in range(3)], axis=1)
    return out, np.linalg.norm(X, axis=-1), [b[i + 1] - b[i] for i in range(3)]


def bands_f32_fft(g32, N, sr, idx):
    """The reference's arithmetic with an f32 FFT (scipy's, in place of rustfft): f32 |.| * scale, axes merged (x + y) + z per bin, bins
    summed in order."""
    xw = _windows(g32, N, idx).transpose(0, 2, 1)
    X = scipy.fft.fft(xw, axis=-1)
    assert X.dtype == np.complex64
    mag = (np.abs(_half_pairs(X, N)).astype(F32) * F32(scale_f32(N))).astype(F32)
    merged = (mag[:, 0] + mag[:, 1]) + mag[:, 2]
    b = [0, map_to_bin(N, sr, 2.0), map_to_bin(N, sr, 30.0), map_to_bin(N, sr, 2000.0)]
    out = np.zeros((merged.shape[0], 3), F32)
    for i in range(3):
        if b[i + 1] > b[i]:
            out[:, i] = np.cumsum(merged[:, b[i]:b[i + 1]], axis=1, dtype=F32)[:, -1]
    return out


_filter_max = {}


def bluestein_m(N):
    return 1 << (2 * N - 2).bit_length()


def filter_max(N):
    """max_k |FFT_M(b)[k]| for Bluestein's filter b (conj of the chirp exp(-i pi n^2 / N), wrapped into M)."""
    if N not in _filter_max:
        M = bluestein_m(N)
        m = np.arange(N, dtype=np.int64)
        ph = (m * m % (2 * N)) / N
        c = np.cos(np.pi * ph) + 1j * np.sin(np.pi * ph)                   # conj(exp(-i pi ph))
        b = np.zeros(M, complex); b[:N] = c; b[M - N + 1:] = c[1:][::-1]
        _filter_max[N] = float(np.abs(np.fft.fft(b)).max())
    return _filter_max[N]


def eps_fft(N):
    """ℓ2 relative error bound of the f32 Bluestein DFT: ‖ΔX‖₂ <= eps · ‖X‖₂ (DESIGN.md §7)."""
    M = bluestein_m(N)
    L = int(math.log2(M))
    eta = 7.0 * U                                                           # twiddle error + complex butterfly (Higham Thm 24.2)
    return filter_max(N) / math.sqrt(N) * (10.0 * U + 2.0 * L * eta)


def bar(N, norms, exact, nbins):
    """Per window and band: twice the first-order bound on |f32 band - f64 band|."""
    fft_term = scale_f32(N) * math.sqrt(2.0 * N) * eps_fft(N) * np.asarray(norms).sum(axis=1)      # w
    rho = np.array([5.0 * U + (nb + 2) * U / (1.0 - (nb + 2) * U) for nb in nbins])                 # hypot, scale, sums, merge
    return 2.0 * (fft_term[:, None] + rho[None, :] * np.abs(exact))


# ---- decision margins of the selection under the bar ----

def _rank64(lf, mf, hf, low):
    nl = lambda a, t: np.where(a < t, 0.0, a - t)
    if low:
        return (lf + mf) / (1.0 + nl(hf, 450.0) * 0.003)
    return mf / (1.0 + nl(hf, 450.0) * 0.003) / (1.0 + nl(lf, 650.0) * 0.003)


def margins(exact, bars, sr, N, target, trim):
    """How far each decision is from flipping when every band moves by its bar (plus the f32 rounding of the band and the rank formula):
    a dict of the smallest margin per kind of decision; every one must be positive for the points to be determined."""
    e = np.asarray(exact, np.float64); d = np.asarray(bars, np.float64) + U * np.abs(e)
    lf, mf, hf = e[:, 0], e[:, 1], e[:, 2]
    n = e.shape[0]
    inf = float("inf")
    out = {}
    mf_hi, mf_lo = mf + d[:, 1], mf - d[:, 1]
    low = bool(np.max(mf, initial=0.0) < 50.0)
    out["mf_max_vs_50"] = (50.0 - np.max(mf_hi, initial=0.0)) if low else (np.max(mf_lo, initial=0.0) - 50.0)
    r = _rank64(lf, mf, hf, low)
    if low:
        lo = _rank64(lf - d[:, 0], mf - d[:, 1], hf + d[:, 2], True); hi = _rank64(lf + d[:, 0], mf + d[:, 1], hf - d[:, 2], True)
    else:
        lo = _rank64(lf + d[:, 0], mf - d[:, 1], hf + d[:, 2], False); hi = _rank64(lf - d[:, 0], mf + d[:, 1], hf - d[:, 2], False)
    w = np.maximum(hi - r, r - lo) + 12.0 * U * np.abs(r)
    ratio = STEP / sr
    time = np.arange(n) * ratio
    inside = np.zeros(n, bool)
    for a, b in np.asarray(trim, np.float64).reshape(-1, 2):
        inside |= (time >= a) & (time <= b)
    total = n * ratio
    if total > 12.0:
        inside &= ~((time < 2.0) | (time >= total - 2.0))
    out["rank_vs_50"] = float(np.min(np.abs(r[inside] - 50.0) - w[inside], initial=inf))
    keep = inside & (r >= 50.0)
    v = np.where(keep, r, 0.0); wv = np.where(keep, w, 0.0)
    radius = as_usize(sr / 16.0 / 2.0 * 8.0)
    # NMS: j (nonzero, < n - 1) against the extremes of its suppressors i in (j - r, j + r]
    top = np.full(n, -inf); top_lo = np.full(n, -inf); top_hi = np.full(n, -inf)
    for dd in range(-radius + 1, radius + 1):
        j = np.arange(max(0, -dd), min(n - 1, n - dd)) if dd else np.zeros(0, int)     # i = j never decides anything
        if j.size:
            top[j] = np.maximum(top[j], v[j + dd])
            top_lo[j] = np.maximum(top_lo[j], v[j + dd] - wv[j + dd]); top_hi[j] = np.maximum(top_hi[j], v[j + dd] + wv[j + dd])
    js = np.nonzero(keep[:-1])[0] if n > 1 else np.zeros(0, int)
    m = np.maximum(top_lo[js] - (v[js] + wv[js]), (v[js] - wv[js]) - top_hi[js])
    out["nms"] = float(np.min(m, initial=inf))
    survive = keep & ~(v < top)
    # segments: the winner against every other survivor of its segment
    seg = (n + target - 1) // target if n else 0
    sm = inf
    for s in range(target):
        start = s * seg; end = min(start + seg, n)
        idx = np.arange(start, end)
        idx = idx[survive[idx]] if idx.size else idx
        if idx.size > 1:
            k = idx[np.argmax(v[idx])]
            others = idx[idx != k]
            sm = min(sm, float((v[k] - wv[k]) - np.max(v[others] + wv[others])))
    out["segment"] = sm
    return out
