"""The visual-features sync search (gf_cuda_sync_costs / gf_cuda_find_sync_offsets, sync_cost_kernel in zoom_kernel.cu): find_offsets
and its calculate_distance (visual_features.rs:9-145), for the "Visual features" offset method and the rolling-shutter estimate.

Without a GPU: the oracle (oracle/gf_oracle_sync.c) equals the second transcription (tests/np_sync.py) bit for bit, over several
lenses, both modes and the search's quirks.  On the GPU: with suppress_rotation set the point path is exact, so every pair's costs and
results equal the oracle's bit for bit; with the rotation on, the device's costs equal costs composed from gf_cuda_undistort_points,
and stay within a stated bar of the oracle's.
"""
import ctypes as C
import os
import subprocess
import warnings

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi
from tests import np_sync, oracle_lib
from tests.test_zoom import _distorting_mesh, _zoom_stab, make_cp

FPS = 30.0
_sync_oracle = None


def _oracle():
    """oracle/libgf_oracle_sync.so (built by __graft_entry__.build(); rebuilt here when its sources are newer, like oracle_lib.load)."""
    global _sync_oracle
    if _sync_oracle is not None:
        return _sync_oracle
    oracle_lib.load()
    path = os.path.join(oracle_lib.ORACLE_DIR, "libgf_oracle_sync.so")
    srcs = ("gf_oracle_sync.c", "gf_oracle_sync.h", "gf_oracle.h", "libgf_oracle.so")
    if not os.path.exists(path) or os.path.getmtime(path) < max(os.path.getmtime(os.path.join(oracle_lib.ORACLE_DIR, f)) for f in srcs):
        subprocess.check_call(["make", "-C", oracle_lib.ORACLE_DIR, "-s", "-f", "sync.mk"])
    lib = C.CDLL(path)
    P = C.POINTER
    lib.gf_oracle_sync_costs.restype = None
    lib.gf_oracle_sync_costs.argtypes = [P(abi.ComputeParams), C.c_int, C.c_int, C.c_double, P(abi.SyncPair), C.c_size_t, C.c_void_p, C.c_void_p,
                                         C.c_size_t, C.c_int, C.c_int, C.c_void_p]
    lib.gf_oracle_find_sync_offsets.restype = C.c_size_t
    lib.gf_oracle_find_sync_offsets.argtypes = [P(abi.ComputeParams), C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int,
                                                P(abi.SyncRange), C.c_size_t, C.c_int, P(abi.SyncResult)]
    _sync_oracle = lib
    return lib


def _lens(name):
    return abi.LENS[name] if name else 0


def oracle_costs(cp, lens, digital, pairs, offsets=None, readouts=None, clear=True, fps=FPS):
    from gyroflow_b200.backend import _sync_pairs
    keep = []
    arr = _sync_pairs(pairs, keep)
    offs = None if offsets is None else np.ascontiguousarray(offsets, np.float64)
    rs = None if readouts is None else np.ascontiguousarray(readouts, np.float64)
    n = len(offs) if offs is not None else len(rs)
    out = np.zeros(n)
    _oracle().gf_oracle_sync_costs(C.byref(cp.c), _lens(lens), _lens(digital), fps, arr, len(pairs), None if offs is None else offs.ctypes.data,
                                   None if rs is None else rs.ctypes.data, n, int(clear), 0, out.ctypes.data)
    return out


def oracle_find(cp, lens, digital, ranges, initial, search, for_rs, fps=FPS):
    from gyroflow_b200.backend import _sync_pairs
    keep = []
    arr = (abi.SyncRange * max(1, len(ranges)))()
    for i, (a, b, pairs) in enumerate(ranges):
        arr[i].from_us, arr[i].to_us = a, b
        arr[i].pairs = _sync_pairs(pairs, keep); arr[i].n_pairs = len(pairs)
    out = (abi.SyncResult * max(1, len(ranges)))()
    n = _oracle().gf_oracle_find_sync_offsets(C.byref(cp.c), _lens(lens), _lens(digital), fps, initial, search, int(for_rs), arr, len(ranges), 0, out)
    return [(out[i].timestamp_ms, out[i].value_ms, out[i].cost) for i in range(n)]


def pairs_at(ts_list, n, w=1920, h=1080, seed=0, shift=(2.5, -1.5), margin=0.1):
    """A matched pair per timestamp (next frame 1 / FPS later): n points inside the frame (`margin` of it left free on every side),
    the second list moved by `shift` plus noise."""
    rng = np.random.default_rng(seed)
    out = []
    for ts in ts_list:
        p1 = (rng.random((n, 2)) * [(1 - 2 * margin) * w, (1 - 2 * margin) * h] + [margin * w, margin * h]).astype(np.float32)
        p2 = (p1 + np.asarray(shift, np.float32) + rng.normal(0, 0.8, (n, 2))).astype(np.float32)
        out.append(((int(ts), p1), (int(ts + round(1e6 / FPS)), p2)))
    return out


def same(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.uint64), np.asarray(b, np.float64).view(np.uint64))


# ---- without a GPU: the oracle against the second transcription ----------------------------------------------------------------------
CPU_LENSES = [("opencv_fisheye", None), ("sony", "digital_stretch"), ("poly3", None), ("gopro", "gopro_warp")]


def _cpu_cp(lens, digital, **kw):
    """Rotation on, rolling shutter, IBIS on frames 0..3 (stabs) and a distorting mesh on frames 0 and 2."""
    stabs = _zoom_stab(4, 1080)
    meshes = [_distorting_mesh(1920, 1080, True, 7), None, _distorting_mesh(1920, 1080, False, 7)]
    return make_cp(lens=lens, digital=digital, camera_stab=stabs, distorting_meshes=meshes, **kw), stabs, meshes


@pytest.mark.parametrize("lens,digital", CPU_LENSES)
def test_costs_oracle_matches_second_restatement(lens, digital):
    """Costs of offsets and of readout times (negative ones included): pairs of n = 1, 9, 10, 11 points (k = 0, 8, 9, 9), an empty
    pair list, and timestamps whose frame is negative (it wraps and finds no IBIS entry, no mesh) next to frames 0..3 that have them."""
    cp, stabs, meshes = _cpu_cp(lens, digital)
    pairs = [pairs_at([10_000.0], 1, seed=1)[0], pairs_at([40_000.0], 9, seed=2)[0], pairs_at([70_000.0], 10, seed=3)[0],
             pairs_at([20_000.0], 11, seed=4)[0]]
    offsets = [-60.0, -12.5, 0.0, 0.37, 25.0, 61.0]          # 61 ms: every timestamp lands before frame 0
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for sel in (pairs, pairs[:1], []):
            want = np_sync.sync_costs(cp, sel, offsets, None, FPS, lens, digital, stabs, meshes)
            assert same(oracle_costs(cp, lens, digital, sel, offsets), want), (sel and len(sel), oracle_costs(cp, lens, digital, sel, offsets), want)
        readouts = [-20.0, -3.25, 0.0, 8.5, 33.0]
        want = np_sync.sync_costs(cp, pairs, None, readouts, FPS, lens, digital, stabs, meshes)
        got = oracle_costs(cp, lens, digital, pairs, readouts=readouts, clear=False)
        assert same(got, want), (got, want)
        assert len(set(want)) > 2                              # the costs do depend on the candidate
    assert same(oracle_costs(cp, lens, digital, pairs[:1], offsets), np.zeros(len(offsets)))      # n = 1: k = 0


def test_find_offsets_oracle_matches_second_restatement():
    """find_offsets, both modes: a range with pairs, an empty range (every cost 0: the last coarse candidate + 0.99 wins, a tie), a
    range whose pairs do not depend on the offset (ties with a non-zero cost), fractional and empty search sizes, fps above 1000 for
    the rolling-shutter estimate, and the 0.9 search-size window: the sweep keeps some results and drops others."""
    lens, digital = "opencv_fisheye", None
    cp, stabs, meshes = _cpu_cp(lens, digital)
    still = make_cp(lens=lens, frame_readout_time_ms=0.0); still.c.suppress_rotation = 1
    ranges = [(0, 200_000, pairs_at([40_000.0, 90_000.0], 10, seed=7)), (200_000, 250_001, [])]
    kept = dropped = 0
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        # (-14.1, 2) lands 1.8 ms or more from the initial offset and is dropped, (-13.9, 2) 1.79 ms from it and kept
        for initial, search in ((0.0, 3.0), (5.0, 2.5), (-20.0, 1.5), (-14.1, 2.0), (-13.9, 2.0), (30.0, 0.5), (0.0, -1.0)):
            want = np_sync.find_offsets(cp, ranges, initial, search, False, FPS, lens, digital, stabs, meshes)
            got = oracle_find(cp, lens, digital, ranges, initial, search, False)
            assert got == want and all(same(a, b) for a, b in zip(got, want)), (initial, search, got, want)
            steps = int(search) if search > 0 else 0
            kept += len(got); dropped += 2 * (steps > 0) - len(got)
            if steps:
                last = initial + (-(search / 2.0) + (steps - 1))
                empty = [r for r in got if r[0] == (200_000 + 50_001 / 2.0) / 1000.0]
                assert all(r[1] == last - 1.0 + 199 * 0.01 and r[2] == 0.0 for r in empty)
        assert kept and dropped, (kept, dropped)
        tie = [(0, 100_000, pairs_at([30_000.0], 10, seed=9))]
        want = np_sync.find_offsets(still, tie, 0.0, 4.0, False, FPS, lens, None)
        got = oracle_find(still, lens, None, tie, 0.0, 4.0, False)
        assert got == want and len(got) == 1 and got[0][1] == (0.0 + (-2.0 + 3.0)) - 1.0 + 199 * 0.01 and got[0][2] > 0, (got, want)
        rs_cp = make_cp(lens=lens, camera_stab=stabs)
        for fps in (400.0, 1001.0):
            want = np_sync.find_offsets(rs_cp, ranges[:1], 0.0, 0.0, True, fps, lens, None, stabs)
            got = oracle_find(rs_cp, lens, None, ranges[:1], 0.0, 0.0, True, fps=fps)
            assert got == want and len(got) == (1 if fps < 1000 else 0), (fps, got, want)


def test_struct_layout():
    """gf_sync_pair / gf_sync_range / gf_sync_result have the same size in abi.py and in the library."""
    lib = abi.load_library()
    for which, cls, size in ((13, abi.SyncPair, 40), (14, abi.SyncRange, 32), (15, abi.SyncResult, 24)):
        assert lib.gf_abi_struct_size(which) == C.sizeof(cls) == size, (which, cls.__name__)
    assert abi.SyncPair.n.offset == 32 and abi.SyncRange.pairs.offset == 16 and abi.SyncResult.cost.offset == 16


# ---- on the GPU ------------------------------------------------------------------------------------------------------------------------
def _gpu_pairs(n_pairs, n, seed=0, t0=20_000.0, margin=0.1):
    return pairs_at([t0 + 45_000.0 * i for i in range(n_pairs)], n, seed=seed, margin=margin)


@pytest.mark.gpu
def test_rotation_free_pairs_match_oracle():
    """suppress_rotation set, so the point path is exact: for every lens pair of the point path, both modes, every candidate's cost and
    every result equals the oracle bit for bit.  IBIS with rolling shutter and distorting meshes make the costs depend on the frame,
    and early timestamps give negative frames."""
    from tests.test_point_matrix import POINT_PAIRS
    stabs = _zoom_stab(6, 1080)
    meshes = [_distorting_mesh(1920, 1080, True, 9), None, _distorting_mesh(1920, 1080, False, 9)]
    ranges = [(0, 150_000, _gpu_pairs(3, 150, seed=1)), (150_000, 400_000, _gpu_pairs(2, 11, seed=2, t0=180_000.0)), (400_000, 500_000, [])]
    offsets = np.concatenate([np.arange(-80.0, 80.0, 0.73), [0.0]])
    readouts = np.arange(-40.0, 40.0, 1.37)
    failures = []
    for lens, digital in POINT_PAIRS:
        cp = make_cp(lens=lens, digital=digital, camera_stab=stabs, distorting_meshes=meshes, gyro_offset_ms=3.5)
        cp.c.suppress_rotation = 1
        dg = g.DeviceGyro(cp)
        try:
            for clear, rs in ((True, None), (False, readouts)):
                pairs = ranges[0][2] + ranges[1][2]
                cand = offsets if rs is None else None
                got = dg.sync_costs(lens, digital, FPS, pairs, offsets_ms=cand, readout_ms=rs, clear_offsets=clear)
                want = oracle_costs(cp, lens, digital, pairs, cand, rs, clear)
                if not same(got, want):
                    failures.append("%s costs clear=%d: %d of %d differ" % ((lens, digital), clear, int((got != want).sum()), got.size))
            for for_rs in (False, True):
                got = dg.find_sync_offsets(lens, digital, FPS, ranges, 4.0, 12.0, for_rs=for_rs)
                want = oracle_find(cp, lens, digital, ranges, 4.0, 12.0, for_rs)
                if not (got == want and all(same(a, b) for a, b in zip(got, want))):
                    failures.append("%s find for_rs=%d: %r != %r" % ((lens, digital), for_rs, got, want))
        finally:
            dg.close()
    assert not failures, failures


def _bar(cp, lens, digital, pairs, offs, rs, fps=FPS):
    """The bar of one candidate against the oracle, from the point path's 2e-3 px bar per coordinate with the rotation on: a distance
    (dx^2 + dy^2) moves by at most 2 * 4e-3 * (|dx| + |dy|) + 2 * (4e-3)^2 when both points move by 2e-3 px per coordinate, and by 1 more
    for the truncation to an integer; the sum of a pair's k smallest distances moves by at most k times the largest such move.  The
    points keep a margin of a tenth of the frame, far from the inside test's edges, so no point pair changes sides."""
    from tests.test_point_matrix import oracle_points
    c = cp.c
    saved = c.frame_readout_time
    if rs is not None:
        c.frame_readout_time = rs
    total = 0.0
    try:
        for (ts, p1), (nts, p2) in pairs:
            t1, t2 = ts / 1000.0 - offs, nts / 1000.0 - offs
            u1 = oracle_points(cp, lens, digital, p1, t1, np_sync.frame_at_timestamp(t1, fps), 1.0, False)
            u2 = oracle_points(cp, lens, digital, p2, t2, np_sync.frame_at_timestamp(t2, fps), 1.0, False)
            inside = ((u1 > 0) & (u1 < [c.width, c.height]) & (u2 > 0) & (u2 < [c.width, c.height])).all(axis=1)
            l1 = np.abs(u2 - u1).sum(axis=1)[inside]
            if l1.size:
                total += int(l1.size * 0.9) * (1.0 + 8e-3 * float(l1.max()) + 2 * 16e-6)
    finally:
        c.frame_readout_time = saved
    return total


@pytest.mark.gpu
def test_rotation_on_matches_undistort_points_and_stays_near_oracle():
    """Rotation, rolling shutter, IBIS and per-frame lens data: gf_cuda_sync_costs equals the costs composed on the host from
    gf_cuda_undistort_points of the same lists, timestamps and frames, bit for bit.  Without per-frame lens data (the oracle has none),
    every cost stays within _bar of the oracle's, and the oracle's cost at the device's chosen offset within twice that bar of the
    oracle's minimum (the device's minimum is at most one bar above the oracle's, the oracle's cost there at most one bar above it)."""
    from tests.test_point_matrix import LENS_A, LENS_B
    lens = "opencv_fisheye"
    stabs = _zoom_stab(8, 1080)
    pairs = _gpu_pairs(2, 40, seed=3, t0=40_000.0)
    offsets = np.array([-45.0, -7.25, 0.0, 3.5, 31.0])
    readouts = np.array([-12.0, 0.0, 9.75])
    lens_cp = make_cp(lens=lens, camera_stab=stabs, lens_per_frame=[LENS_A, LENS_B, LENS_A], sync_offsets={0: 2.0, 2_000_000: 6.0})
    dg = g.DeviceGyro(lens_cp)
    plain = make_cp(lens=lens)                 # no sync offsets uploaded: what clear_offsets makes of lens_cp
    plain_cp = make_cp(lens=lens, camera_stab=stabs, lens_per_frame=[LENS_A, LENS_B, LENS_A])
    pdg = g.DeviceGyro(plain_cp)
    try:
        points = lambda d: (lambda pts, t: d.undistort_points(lens, None, pts, t, frame=np_sync.frame_at_timestamp(t, FPS)))
        got = dg.sync_costs(lens, None, FPS, pairs, offsets_ms=offsets, clear_offsets=True)
        want = np_sync.sync_costs(plain_cp, pairs, offsets, None, FPS, lens, None, points=points(pdg))
        assert same(got, want), (got, want)
        got = dg.sync_costs(lens, None, FPS, pairs, readout_ms=readouts, clear_offsets=False)
        want = np_sync.sync_costs(lens_cp, pairs, None, readouts, FPS, lens, None, points=points(dg))
        assert same(got, want), (got, want)
    finally:
        dg.close(); pdg.close()
    del plain
    cp = make_cp(lens=lens, camera_stab=stabs)
    dg = g.DeviceGyro(cp)
    try:
        got = dg.sync_costs(lens, None, FPS, pairs, offsets_ms=offsets)
        want = oracle_costs(cp, lens, None, pairs, offsets)
        bars = np.array([_bar(cp, lens, None, pairs, o, None) for o in offsets])
        assert (np.abs(got - want) <= bars).all(), (got, want, bars)
        ranges = [(0, 200_000, pairs)]
        dev = dg.find_sync_offsets(lens, None, FPS, ranges, 0.0, 20.0)
        ora = oracle_find(cp, lens, None, ranges, 0.0, 20.0, False)
        assert len(dev) == len(ora) == 1
        at_dev = oracle_costs(cp, lens, None, pairs, [dev[0][1]])[0]
        assert at_dev <= ora[0][2] + 2 * _bar(cp, lens, None, pairs, dev[0][1], None), (dev, ora, at_dev)
    finally:
        dg.close()


@pytest.mark.gpu
def test_large_pair_and_chunked_search():
    """A pair of 9000 points (more than the kernel's 8192 shared-memory keys: its keys live in global scratch) and a 5000-candidate
    offset search over 12 pairs (its records take several chunks), bit for bit against the oracle with the rotation suppressed."""
    stabs = _zoom_stab(6, 1080)
    cp = make_cp(lens="sony", camera_stab=stabs, params=dict(lens_correction_amount=0.7))
    cp.c.suppress_rotation = 1
    dg = g.DeviceGyro(cp)
    try:
        big = _gpu_pairs(1, 9000, seed=5, margin=0.0) + _gpu_pairs(1, 300, seed=6, t0=70_000.0)
        offsets = np.array([-70.0, -33.3, 0.0, 12.0, 50.0])
        got = dg.sync_costs("sony", None, FPS, big, offsets_ms=offsets)
        assert same(got, oracle_costs(cp, "sony", None, big, offsets)), got
        ranges = [(0, 600_000, _gpu_pairs(12, 24, seed=8))]
        dev = dg.find_sync_offsets("sony", None, FPS, ranges, 10.0, 5000.0)
        timing = dg.sync_timing()
        assert timing["chunks"] > 2 and timing["device_ms"] > 0.0 and timing["host_record_ms"] > 0.0, timing
        ora = oracle_find(cp, "sony", None, ranges, 10.0, 5000.0, False)
        assert dev == ora and all(same(a, b) for a, b in zip(dev, ora)), (dev, ora)
    finally:
        dg.close()


@pytest.mark.gpu
def test_argument_validation():
    """Refusals before any work, each with GF_ERR_BAD_PARAMS (or UNSUPPORTED_COMBO) and a message: the 2^53 bound on
    sum(n) * (width^2 + height^2), frames above 32768 px, a non-positive or NaN fps, null point lists, search sizes of 1e7 ms or more,
    more than 1e7 readout times, and a lens pair the point path does not compile.  No candidates is not an error."""
    lib = abi.load_library()
    cp = make_cp(w=32768, h=32768)
    dg = g.DeviceGyro(cp)
    try:
        # 2^53 / (2 * 32768^2) = 2^22 points reach the bound exactly
        n = 1 << 22
        pts = np.zeros((n, 2), np.float32)
        pairs = [((0, pts[: n // 2]), (33_333, pts[: n // 2])), ((0, pts[n // 2:]), (33_333, pts[n // 2:]))]
        with pytest.raises(g.GyroflowCoreError) as e:
            dg.sync_costs("opencv_fisheye", None, FPS, pairs, offsets_ms=[0.0])
        assert e.value.code == -1 and "2^53" in str(e.value)
        small = [((0, pts[:8]), (33_333, pts[:8]))]
        assert dg.sync_costs("opencv_fisheye", None, FPS, small, offsets_ms=[]).size == 0
        for fps in (0.0, -30.0, float("nan"), float("inf")):
            with pytest.raises(g.GyroflowCoreError) as e:
                dg.sync_costs("opencv_fisheye", None, fps, small, offsets_ms=[0.0])
            assert e.value.code == -1 and "scaled_fps" in str(e.value)
        with pytest.raises(g.GyroflowCoreError) as e:
            dg.sync_costs("opencv_fisheye", "gopro_warp", FPS, small, offsets_ms=[0.0])
        assert e.value.code == -5
        with pytest.raises(g.GyroflowCoreError) as e:
            dg.find_sync_offsets("opencv_fisheye", None, FPS, [(0, 1, small)], 0.0, 1e7)
        assert e.value.code == -1 and "search_size" in str(e.value)
        with pytest.raises(g.GyroflowCoreError) as e:
            dg.estimate_rolling_shutter("opencv_fisheye", None, 1e-4, [(0, 1, small)])
        assert e.value.code == -1 and "readout" in str(e.value)
        bad = (abi.SyncPair * 1)()
        bad[0].n = 4
        offs = np.zeros(1); out = np.zeros(1)
        rc = lib.gf_cuda_sync_costs(dg._h, C.byref(cp.c), 1, 0, FPS, bad, 1, offs.ctypes.data, None, 1, 1, out.ctypes.data, None)
        assert rc == -1 and b"null point list" in lib.gf_cuda_last_error(None)
    finally:
        dg.close()
    big = make_cp(w=32769, h=64)
    dg = g.DeviceGyro(big)
    try:
        with pytest.raises(g.GyroflowCoreError) as e:
            dg.sync_costs("opencv_fisheye", None, FPS, [((0, np.ones((2, 2), np.float32)), (1, np.ones((2, 2), np.float32)))], offsets_ms=[0.0])
        assert e.value.code == -1 and "32768" in str(e.value)
    finally:
        dg.close()
