"""The automatic choice of sync points (gf_optimal_sync_sizes / gf_optimal_sync_select / gf_cuda_optimal_sync_points, optimal_sync.cu):
OptimSync::new + run (optimsync.rs:30-225).

Without a GPU: the oracle (oracle/gf_oracle_optsync.c) equals the second transcription (tests/np_optsync.py) bit for bit on the
resampling, blackman and the selection; the library's selection (O(windows) NMS) equals the oracle's literal double loop bit for bit;
the sizes query agrees with the transcription and refuses each documented case; an f32 FFT's band energies lie within the bar.
On the GPU: the resampling hook equals the oracle bit for bit, the band energies lie within the bar of the f64 oracle, NaN and Inf
samples give NaN in exactly their windows, the returned rank and points are the selection of the returned band energies, and on
engineered clips whose every decision clears the bar the points equal the f64 oracle's.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi
from tests import np_optsync as npo
from tests import oracle_lib

F32 = np.float32
_lib_o = None


def _oracle():
    """oracle/libgf_oracle_optsync.so (built by __graft_entry__.build(); rebuilt here when its source is newer)."""
    global _lib_o
    if _lib_o is not None:
        return _lib_o
    d = oracle_lib.ORACLE_DIR
    path = os.path.join(d, "libgf_oracle_optsync.so")
    if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(d, "gf_oracle_optsync.c")):
        subprocess.check_call(["make", "-C", d, "-s", "-f", "optsync.mk"])
    lib = C.CDLL(path)
    lib.gf_oracle_optsync_resample.restype = C.c_size_t
    lib.gf_oracle_optsync_resample.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_double), C.c_void_p]
    lib.gf_oracle_optsync_blackman.restype = None
    lib.gf_oracle_optsync_blackman.argtypes = [C.c_size_t, C.c_void_p]
    lib.gf_oracle_optsync_select.restype = C.c_size_t
    lib.gf_oracle_optsync_select.argtypes = [C.c_void_p, C.c_size_t, C.c_double, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                             C.c_void_p, C.POINTER(C.c_double), C.c_void_p, C.c_void_p]
    _lib_o = lib
    return lib


def o_resample(ts, gyro, has=None):
    ts = np.ascontiguousarray(ts, np.float64); gy = np.ascontiguousarray(gyro, np.float64).reshape(-1, 3)
    hg = None if has is None else np.ascontiguousarray(has, np.uint8)
    sr = C.c_double()
    n = _oracle().gf_oracle_optsync_resample(ts.ctypes.data, gy.ctypes.data, None if hg is None else hg.ctypes.data, ts.size, C.byref(sr), None)
    out = np.zeros((n, 3))
    _oracle().gf_oracle_optsync_resample(ts.ctypes.data, gy.ctypes.data, None if hg is None else hg.ctypes.data, ts.size, C.byref(sr), out.ctypes.data)
    return sr.value, out


def o_blackman(N):
    out = np.zeros(N, F32)
    _oracle().gf_oracle_optsync_blackman(N, out.ctypes.data)
    return out


def o_select(bands, sr, N, target, trim):
    b = np.ascontiguousarray(bands, F32).reshape(-1, 3)
    t = np.ascontiguousarray(trim, np.float64).reshape(-1, 2)
    n = b.shape[0]
    pts = np.zeros(max(target, 1)); rank = np.zeros(n, F32); s1 = np.zeros(n, F32); s2 = np.zeros(n, F32); ratio = C.c_double()
    k = _oracle().gf_oracle_optsync_select(b.ctypes.data, n, sr, N, target, t.ctypes.data if t.size else None, t.shape[0], pts.ctypes.data,
                                           rank.ctypes.data, C.byref(ratio), s1.ctypes.data, s2.ctypes.data)
    return pts[:k].copy(), rank, ratio.value


def same_bits(a, b):
    a = np.asarray(a); b = np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def uniform_log(sr_target, seconds, rng=None, amp=20.0):
    """A log at exactly sr_target Hz of samples, so that round(avg_sr) is sr_target for long enough logs."""
    n = int(round(seconds * sr_target)) + 1
    ts = np.arange(n) * (1000.0 / sr_target)
    rng = rng or np.random.default_rng(1)
    return ts, rng.normal(0.0, amp, (n, 3))


def logs():
    rng = np.random.default_rng(7)
    out = {}
    n = 3000
    out["jittered"] = (np.cumsum(rng.uniform(0.5, 1.5, n)) - 0.3, rng.normal(0, 1, (n, 3)), None)
    has = rng.random(n) > 0.2
    out["gaps"] = (np.arange(n) * 1.25 + 0.1, rng.normal(0, 1, (n, 3)), has)
    out["start_above_0"] = (np.arange(n) * 2.0 + 537.25, rng.normal(0, 1, (n, 3)), None)
    out["start_below_0"] = (np.arange(n) * 2.0 - 1234.5, rng.normal(0, 1, (n, 3)), None)
    out["extrapolate"] = (np.concatenate([[0.0, 0.4], 0.4 + np.cumsum(rng.uniform(3.0, 4.0, 200))]), rng.normal(0, 1, (202, 3)), None)
    out["single"] = (np.array([5.0]), np.array([[1.0, 2.0, 3.0]]), None)
    out["two"] = (np.array([0.0, 250.0]), np.array([[1.0, 2.0, 3.0], [4.0, -5.0, 6.0]]), None)
    return out


# ---------------------------------------------------------------- without a GPU

@pytest.mark.parametrize("name", sorted(logs()))
def test_oracle_resample_equals_transcription(name):
    ts, gy, has = logs()[name]
    if ts.size < 2:
        return      # a single sample spans no time: refused by the sizes query (below), nothing to resample
    sr_o, out_o = o_resample(ts, gy, has)
    sr_n, out_n = npo.resample(ts, gy, has)
    assert sr_o == sr_n and same_bits(out_o, out_n)
    assert out_o.shape[0] > 0 or name == "two"


@pytest.mark.parametrize("N", [4, 25, 200, 1999, 8000, 8192])
def test_oracle_blackman_equals_transcription(N):
    assert same_bits(o_blackman(N), npo.blackman(N))


def selection_cases():
    rng = np.random.default_rng(11)
    cases = []
    def add(name, bands, sr, N, target, trim):
        cases.append((name, np.asarray(bands, F32).reshape(-1, 3), sr, N, target, np.asarray(trim, np.float64).reshape(-1, 2)))
    whole = [(-1e9, 1e9)]
    add("random", rng.uniform(0, 400, (3000, 3)), 200.0, 200, 5, whole)
    add("random_big_r", rng.uniform(0, 900, (20000, 3)), 1000.0, 1000, 7, whole)        # r = 250
    add("r0", rng.uniform(0, 400, (500, 3)), 3.9, 4, 3, whole)                          # r = (3.9 / 32 * 8) as usize = 0
    add("tied", np.repeat(rng.integers(0, 4, (400, 1)) * 60.0, 3, axis=1), 200.0, 200, 4, whole)
    add("zero", np.zeros((300, 3)), 200.0, 200, 3, whole)
    b = rng.uniform(40, 400, (600, 3)); b[rng.random(600) < 0.05] = np.nan
    add("nan", b, 200.0, 200, 6, whole)
    b = rng.uniform(40, 400, (600, 3)); b[100:110, 1] = np.nan; b[250, :] = np.nan
    add("nan_in_segment", b, 200.0, 200, 3, whole)
    add("low_motion", rng.uniform(0, 49.9, (700, 3)) * [20, 1, 12], 200.0, 200, 4, whole)
    sr = 200.0; ratio = 16.0 / sr
    add("trim_end_exact", rng.uniform(0, 400, (800, 3)), sr, 200, 4, [(10 * ratio, 123 * ratio), (300 * ratio, 511 * ratio)])
    n12 = int(12.0 / ratio)                                                              # 150 windows: total exactly 12 s
    add("total_12s", rng.uniform(40, 400, (n12, 3)), sr, 200, 3, whole)
    add("total_over_12s", rng.uniform(40, 400, (n12 + 1, 3)), sr, 200, 3, whole)        # a window sits at exactly total - 2
    add("target_gt_windows", rng.uniform(40, 400, (7, 3)), sr, 200, 20, whole)
    add("len_not_divisible", rng.uniform(40, 400, (1001, 3)), sr, 200, 7, whole)
    add("empty", np.zeros((0, 3)), sr, 200, 3, whole)
    add("one", [[1.0, 300.0, 2.0]], sr, 200, 3, whole)
    add("no_trim", rng.uniform(40, 400, (100, 3)), sr, 200, 3, np.zeros((0, 2)))
    add("inf", np.where(rng.random((300, 3)) < 0.02, np.inf, rng.uniform(40, 400, (300, 3))), sr, 200, 4, whole)
    return cases


@pytest.mark.parametrize("case", selection_cases(), ids=lambda c: c[0])
def test_selection_oracle_transcription_library(case):
    name, bands, sr, N, target, trim = case
    pts_o, rank_o, ratio_o = o_select(bands, sr, N, target, trim)
    pts_n, rank_n, ratio_n = npo.select(bands, sr, N, target, trim)
    pts_l, rank_l, ratio_l = g.optimal_sync_select(bands, sr, N, target, trim)
    assert same_bits(pts_o, pts_n) and same_bits(rank_o, rank_n) and ratio_o == ratio_n
    assert same_bits(pts_o, pts_l) and same_bits(rank_o, rank_l) and ratio_o == ratio_l
    if name in ("random", "random_big_r", "tied", "nan", "len_not_divisible"):
        assert pts_o.size > 0


def test_selection_exercises_its_branches():
    """The engineered cases reach what they are named after."""
    cases = {c[0]: c for c in selection_cases()}
    _, b, sr, N, t, trim = cases["low_motion"]
    assert npo.ranks(b)[1] and not npo.ranks(cases["random"][1])[1]
    _, b, sr, N, t, trim = cases["total_over_12s"]
    ratio = 16.0 / sr
    total = b.shape[0] * ratio
    assert total > 12.0 and any(i * ratio == total - 2.0 for i in range(b.shape[0]))
    assert cases["total_12s"][1].shape[0] * ratio == 12.0
    _, b, sr, N, t, trim = cases["trim_end_exact"]
    assert 123 * (16.0 / sr) == trim[0, 1]


def test_sizes_agree_and_refuse():
    for name, (ts, gy, has) in logs().items():
        if ts.size < 2:
            continue
        sr, N, nr, nw = npo.sizes(ts, has)
        if N < 4 or N > 8192:
            continue
        assert g.optimal_sync_sizes(ts, has) == (sr, N, nr, nw), name
    for sr_t in (200, 1999, 8000, 8192):
        ts, _ = uniform_log(sr_t, 3.0)
        got = g.optimal_sync_sizes(ts)
        assert got == npo.sizes(ts) and got[1] == sr_t and got[3] > 0
    lib = abi.load_library()
    def rc(ts, has=None):
        ts = np.ascontiguousarray(ts, np.float64)
        hg = None if has is None else np.ascontiguousarray(has, np.uint8)
        return lib.gf_optimal_sync_sizes(ts.ctypes.data, None if hg is None else hg.ctypes.data, ts.size, None, None, None, None)
    assert rc(np.zeros(0)) == -8                                     # empty log: new returns None
    assert rc([5.0]) == -1 and rc([3.0, 3.0, 3.0]) == -1            # no duration
    assert rc([0.0, np.nan, 2.0]) == -1 and rc([0.0, 2.0, 1.0, 3.0]) == -1
    assert rc(np.arange(10) * 1000.0, np.zeros(10)) == -1            # no gyro sample
    assert rc(np.arange(4) * 1000.0) == -1                           # 4 / 3 s -> N = 1
    assert rc(np.arange(101) * (1000.0 / 3.4)) == -1                 # round(3.434) = 3
    assert rc(np.arange(101) * (1000.0 / 3.6)) == 0                  # round(3.636) = 4
    assert rc(np.arange(20001) * (1000.0 / 8192.0)) == 0
    assert rc(np.arange(20001) * (1000.0 / 8193.0)) == -1           # N = 8193
    assert lib.gf_optimal_sync_select(None, 0, 200.0, 200, 0, None, 0, np.zeros(1).ctypes.data, C.byref(C.c_size_t()), None, None) == -1


@pytest.mark.parametrize("N", [200, 1999, 8000])
def test_f32_fft_within_bar(N):
    """An f32 FFT with the reference's band arithmetic (scipy's, as rustfft would be) lies within the bar of the f64 spectra."""
    ts, gy = uniform_log(N, 4.0, np.random.default_rng(N))
    sr, g64 = npo.resample(ts, gy)
    assert int(npo.round_half_away(sr)) == N
    g32 = g64.astype(F32)
    nw = (g32.shape[0] - N) // 16 + 1
    idx = np.linspace(0, nw - 1, 12).astype(int)
    ex, norms, nb = npo.bands_f64(g32, N, sr, idx)
    f32 = npo.bands_f32_fft(g32, N, sr, idx)
    bar = npo.bar(N, norms, ex, nb)
    ratio = np.abs(f32.astype(np.float64) - ex) / bar
    assert np.all(ratio <= 1.0), ratio.max()
    print("N=%d: scipy f32 vs f64, worst error %.3g of the bar, worst relative %.3g" % (N, ratio.max(), (np.abs(f32 - ex) / ex).max()))


# ---------------------------------------------------------------- on the GPU

def _device_bands(ts, gy, has=None, target=3, trim=((-1e9, 1e9),)):
    return g.optimal_sync_points(ts, gy, has, target, trim)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(logs()) + ["million"])
def test_gpu_resample_bit_exact(name):
    if name == "million":
        rng = np.random.default_rng(3)
        n = 1_000_000
        ts = np.cumsum(rng.uniform(0.1, 0.15, n)) + 17.0; gy = rng.normal(0, 3, (n, 3)); has = rng.random(n) > 0.01
    else:
        ts, gy, has = logs()[name]
    if ts.size < 2:
        with pytest.raises(g.GyroflowCoreError):        # a single sample spans no time
            g.selftest_optimal_sync_resample(ts, gy, has)
        return
    want = o_resample(ts, gy, has)[1].astype(F32)
    got = g.selftest_optimal_sync_resample(ts, gy, has)
    assert same_bits(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [4, 25, 200, 1000, 1999, 2000, 4096, 8000, 8192])
def test_gpu_bands_within_bar(N):
    rng = np.random.default_rng(100 + N)
    seconds = max(3.0, 40.0 / N)
    ts, _ = uniform_log(N, seconds)
    n = ts.size
    t = ts / 1000.0
    gy = np.stack([30 * np.sin(2 * np.pi * 1.3 * t) + rng.normal(0, 5, n), 20 * np.sin(2 * np.pi * 7.0 * t) + rng.normal(0, 5, n),
                   rng.normal(0, 10, n)], axis=1)
    sr, NN, nr, nw = g.optimal_sync_sizes(ts)
    assert NN == N and nw > 0
    pts, rank, ratio, bands = _device_bands(ts, gy)
    g32 = o_resample(ts, gy)[1].astype(F32)
    idx = np.unique(np.linspace(0, nw - 1, min(nw, 24)).astype(int))
    ex, norms, nb = npo.bands_f64(g32, N, sr, idx)
    bar = npo.bar(N, norms, ex, nb)
    err = np.abs(bands[idx].astype(np.float64) - ex)
    frac = err / np.where(bar > 0, bar, 1.0)
    assert np.all(err <= bar), frac.max()
    print("N=%d: worst device error %.3g of the bar (eps %.3g)" % (N, frac.max(), npo.eps_fft(N)))


@pytest.mark.gpu
def test_gpu_nan_inf_windows():
    N = 200
    ts, gy = uniform_log(N, 20.0)
    gy[1000, 0] = np.nan; gy[2500, 2] = np.inf; gy[3100, 1] = -np.inf
    res = g.selftest_optimal_sync_resample(ts, gy)
    bad = ~np.isfinite(res).all(axis=1)
    pts, rank, ratio, bands = _device_bands(ts, gy)
    nw = bands.shape[0]
    has_bad = np.array([bad[w * 16:w * 16 + N].any() for w in range(nw)])
    assert has_bad.any() and (~has_bad).any()
    assert np.isnan(bands[has_bad]).all() and np.isfinite(bands[~has_bad]).all()


@pytest.mark.gpu
def test_gpu_selection_of_returned_bands():
    rng = np.random.default_rng(5)
    for N, sec, target, trim in ((200, 90.0, 5, [(-1e9, 1e9)]), (1000, 40.0, 3, [(3.0, 20.0), (25.0, 30.0)])):
        ts, gy = uniform_log(N, sec, rng, amp=40.0)
        sr = g.optimal_sync_sizes(ts)[0]
        pts, rank, ratio, bands = _device_bands(ts, gy, None, target, trim)
        pl, rl, al = g.optimal_sync_select(bands, sr, N, target, trim)
        po, ro, ao = o_select(bands, sr, N, target, trim)
        assert same_bits(pts, pl) and same_bits(rank, rl) and ratio == al
        assert same_bits(pts, po) and same_bits(rank, ro) and ratio == ao


def engineered_clip(N, seconds, bursts, rng, base=1.0):
    """Gyro at N Hz: noise of `base` deg/s, plus bursts (t0, t1, f_hz, amp) whose amplitude ramps up over the burst."""
    ts, _ = uniform_log(N, seconds)
    t = ts / 1000.0
    gy = rng.normal(0, base, (ts.size, 3))
    for t0, t1, f, a in bursts:
        m = (t >= t0) & (t < t1)
        env = a * (0.5 + 0.5 * (t[m] - t0) / (t1 - t0))
        gy[m, 0] += env * np.sin(2 * np.pi * f * t[m])
        gy[m, 1] += 0.6 * env * np.cos(2 * np.pi * 1.7 * f * t[m])
    return ts, gy


def clips():
    rng = np.random.default_rng(2024)
    c = {}
    c["bursts"] = engineered_clip(200, 60.0, [(8, 13, 5.0, 200.0), (30, 33, 9.5, 320.0), (45, 50, 4.5, 170.0)], rng, base=0.3) + (3, [(-1e9, 1e9)])
    c["low_motion"] = engineered_clip(200, 40.0, [(10, 14, 0.5, 3.0), (25, 28, 0.6, 2.0)], rng, base=0.05) + (2, [(-1e9, 1e9)])
    c["trim"] = engineered_clip(400, 50.0, [(6, 9, 6.0, 250.0), (20, 24, 8.0, 300.0), (35, 39, 5.0, 200.0)], rng) + (3, [(0.0, 15.0), (30.0, 45.0)])
    c["short_12s"] = engineered_clip(200, 11.0, [(3, 6, 6.0, 200.0)], rng) + (2, [(-1e9, 1e9)])
    c["over_12s_edges"] = engineered_clip(200, 20.0, [(0.5, 2.5, 6.0, 400.0), (9, 12, 7.0, 200.0), (17.5, 19.5, 6.0, 400.0)], rng) + (3, [(-1e9, 1e9)])
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bursts", "low_motion", "trim", "short_12s", "over_12s_edges"])
def test_gpu_points_equal_f64_oracle(name):
    ts, gy, target, trim = clips()[name]
    sr, N, nr, nw = g.optimal_sync_sizes(ts)
    g32 = o_resample(ts, gy)[1].astype(F32)
    ex, norms, nb = npo.bands_f64(g32, N, sr, np.arange(nw))
    bar = npo.bar(N, norms, ex, nb)
    m = npo.margins(ex, bar, sr, N, target, trim)
    assert min(m.values()) > 0, m                      # every decision clears the bar: the points are determined
    want, _, _ = o_select(ex.astype(F32), sr, N, target, trim)
    pts, rank, ratio, bands = _device_bands(ts, gy, None, target, trim)
    assert np.all(np.abs(bands - ex) <= bar)
    assert same_bits(pts, want), (pts, want)
    assert pts.size > 0 and npo.ranks(bands)[1] == (name == "low_motion")
    print(name, "points", pts, "margins", m)


@pytest.mark.gpu
def test_gpu_shorter_than_one_window():
    ts, gy = uniform_log(200, 0.5)
    sr, N, nr, nw = g.optimal_sync_sizes(ts)
    assert nw == 0 and nr > 0
    pts, rank, ratio, bands = _device_bands(ts, gy)
    assert pts.size == 0 and rank.size == 0 and bands.shape == (0, 3) and ratio == 16.0 / sr


@pytest.mark.gpu
def test_gpu_ten_minutes_8khz():
    rng = np.random.default_rng(8000)
    N = 8000
    ts, gy = engineered_clip(N, 600.0, [(100, 110, 6.0, 200.0), (300, 305, 12.0, 250.0), (480, 490, 4.0, 150.0)], rng)
    sr, NN, nr, nw = g.optimal_sync_sizes(ts)
    assert NN == N and nw > 290_000
    pts, rank, ratio, bands = _device_bands(ts, gy, None, 3)
    assert rank.size == nw and np.isfinite(bands).all() and pts.size > 0
    idx = np.sort(np.random.default_rng(1).choice(nw, 1000, replace=False))
    g32 = o_resample(ts, gy)[1].astype(F32)
    worst = 0.0
    for part in np.array_split(idx, 10):
        ex, norms, nb = npo.bands_f64(g32, N, sr, part)
        bar = npo.bar(N, norms, ex, nb)
        err = np.abs(bands[part].astype(np.float64) - ex)
        assert np.all(err <= bar)
        worst = max(worst, float((err / bar).max()))
    print("10 min at 8 kHz: %d windows, worst error %.3g of the bar over 1000 windows" % (nw, worst))


@pytest.mark.gpu
def test_gpu_refusals_before_device_work():
    """Each refusal comes back with its code and no device work: the call on an invalid device ordinal still returns the refusal."""
    lib = abi.load_library()
    out = np.zeros(8); npt = C.c_size_t(); ratio = C.c_double()
    def rc(ts, gy, target=3, device=0, has=None):
        ts = np.ascontiguousarray(ts, np.float64); gy = np.ascontiguousarray(gy, np.float64).reshape(-1, 3)
        hg = None if has is None else np.ascontiguousarray(has, np.uint8)
        return lib.gf_cuda_optimal_sync_points(device, ts.ctypes.data, gy.ctypes.data, None if hg is None else hg.ctypes.data, ts.size, target,
                                               None, 0, out.ctypes.data, C.byref(npt), None, None, C.byref(ratio), None)
    ok_ts, ok_gy = uniform_log(200, 3.0)
    bad_dev = 1 << 20
    assert rc(ok_ts, ok_gy, target=0, device=bad_dev) == -1
    assert rc(np.zeros(0), np.zeros((0, 3)), device=bad_dev) == -8
    assert rc([5.0], [[1, 2, 3]], device=bad_dev) == -1
    assert rc([0.0, np.nan, 2.0], np.zeros((3, 3)), device=bad_dev) == -1
    assert rc([0.0, 2.0, 1.0], np.zeros((3, 3)), device=bad_dev) == -1
    assert rc(np.arange(4) * 1000.0, np.zeros((4, 3)), device=bad_dev) == -1
    assert rc(np.arange(10) * 1000.0, np.zeros((10, 3)), device=bad_dev, has=np.zeros(10)) == -1
    assert rc(np.arange(20001) * (1000.0 / 8193.0), np.zeros((20001, 3)), device=bad_dev) == -1
    # a log shorter than one window launches nothing either
    short_ts, short_gy = uniform_log(200, 0.5)
    assert rc(short_ts, short_gy, device=bad_dev) == 0 and npt.value == 0
    # and a valid call on the device ordinal fails as a CUDA error only once there is work
    assert rc(ok_ts, ok_gy, device=bad_dev) == -6
    assert rc(ok_ts, ok_gy) == 0
