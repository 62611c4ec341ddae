"""The sync cost's k-smallest selection (sync_select_add in gyroflow_b200/csrc/sync_select.cuh, run by sync_cost_kernel) on keys built to
reach every part of its radix select, each result exact against a plain integer reference: sort the valid keys, sum the
k = int(m * 0.9) smallest (visual_features.rs:69-82).

Without a GPU: the engineered point lists really produce the key distributions the GPU tests rely on (keys of every byte, ties across
the k-th key, keys near 2^31, a job just under the 2^53 bound), and the oracle's costs equal the integer reference on keys built from
the oracle's own points.  On the GPU: gf_cuda_selftest_sync_select on raw keys, and gf_cuda_sync_costs / gf_cuda_find_sync_offsets on
the engineered lists, against the reference on keys built from gf_cuda_undistort_points (rotation on) and against the oracle (rotation
suppressed, where the point path is exact).

Counting the keys <= T instead of < T in the final sum gives the same total (the tie term (k - count) * T makes up for it), so no test
can tell those two apart.  A pass-1 or pass-2 mask one byte too wide or too narrow, a prefix or rank left unchanged in pass 1 or 2, or
a dropped tie term each fails at least one test here.
"""
import functools

import numpy as np
import pytest

import gyroflow_b200 as g
from tests import np_sync
from tests.test_point_matrix import oracle_points
from tests.test_sync_offsets import FPS, oracle_costs, oracle_find, same
from tests.test_zoom import _zoom_stab, make_cp

NO_KEY = 0xFFFFFFFF
SMEM_KEYS = 8192                       # SYNC_SMEM_KEYS: larger groups keep their keys in global scratch
F32 = np.float32


# ---- the reference -------------------------------------------------------------------------------------------------------------------
def k_of(m):
    return int(m * 0.9)                # (len as f64 * 0.9) as usize


def select_sum(keys):
    """The sum of the k smallest valid keys, as a Python integer."""
    keys = np.asarray(keys, np.uint64)
    valid = np.sort(keys[keys != NO_KEY])
    return int(valid[:k_of(valid.size)].sum(dtype=np.uint64))


def kth(keys):
    """(k, the k-th smallest valid key T, count of valid keys < T, count == T); T None when k = 0."""
    keys = np.asarray(keys, np.uint64)
    valid = np.sort(keys[keys != NO_KEY])
    k = k_of(valid.size)
    if k == 0:
        return 0, None, 0, 0
    t = int(valid[k - 1])
    return k, t, int((valid < t).sum()), int((valid == t).sum())


def pair_keys(points, pair, off, w, h, fps=FPS):
    """The keys of one pair at offset `off`, as sync_cost_kernel builds them: points(pts, timestamp_ms, frame) gives the undistorted
    (n, 2) float32 points; a point pair inside the frame gives trunc(dx^2 + dy^2) in f32, any other NO_KEY."""
    (ts, p1), (nts, p2) = pair
    if len(p1) == 0:
        return np.zeros(0, np.uint64)
    t1, t2 = ts / 1000.0 - off, nts / 1000.0 - off
    u1 = np.asarray(points(np.asarray(p1, F32), t1, np_sync.frame_at_timestamp(t1, fps)), F32)
    u2 = np.asarray(points(np.asarray(p2, F32), t2, np_sync.frame_at_timestamp(t2, fps)), F32)
    fw, fh = F32(w), F32(h)
    with np.errstate(invalid="ignore", over="ignore"):
        inside = ((u1[:, 0] > 0) & (u1[:, 0] < fw) & (u1[:, 1] > 0) & (u1[:, 1] < fh) &
                  (u2[:, 0] > 0) & (u2[:, 0] < fw) & (u2[:, 1] > 0) & (u2[:, 1] < fh))
        d = u2 - u1
        dist = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]                  # f32, no contraction
    keys = np.full(len(p1), NO_KEY, np.uint64)
    keys[inside] = dist[inside].astype(np.uint64)
    return keys


def exact_costs(points, pairs, offsets, w, h):
    """Every offset's cost from the integer reference; the points of pairs with the same two timestamps go through `points` together."""
    groups = {}
    for (ts, p1), (nts, p2) in pairs:
        groups.setdefault((ts, nts), []).append((np.asarray(p1, F32).reshape(-1, 2), np.asarray(p2, F32).reshape(-1, 2)))
    out = []
    for o in offsets:
        total = 0
        for (ts, nts), lists in groups.items():
            keys = pair_keys(points, ((ts, np.concatenate([a for a, _ in lists])), (nts, np.concatenate([b for _, b in lists]))), o, w, h)
            for part in np.split(keys, np.cumsum([len(a) for a, _ in lists])[:-1]):
                total += select_sum(part)
        out.append(float(total))
    return np.array(out)


def oracle_pts(cp, lens, digital=None):
    return lambda pts, t, frame: oracle_points(cp, lens, digital, pts, t, frame, 1.0, False)


def device_pts(dg, lens, digital=None):
    return lambda pts, t, frame: dg.undistort_points(lens, digital, pts, t, frame=frame)


# ---- the engineered point lists --------------------------------------------------------------------------------------------------------
W4K, H4K, LENS4K = 3840, 2160, "opencv_fisheye"
TS = 40_000                          # every pair's first timestamp (us); the next frame 1 / FPS later
NTS = TS + round(1e6 / FPS)
OFFSETS = np.array([-21.5, -3.0, 0.0, 7.25, 18.0])


def cp_4k(suppress):
    cp = make_cp(w=W4K, h=H4K, lens=LENS4K, camera_stab=_zoom_stab(4, H4K))
    cp.c.suppress_rotation = int(suppress)
    return cp


@functools.lru_cache(maxsize=None)
def _visible_pool(suppress):
    """Distorted points of a 4K fisheye frame whose undistorted position lies at least 8 px inside the frame at both timestamps of every
    offset in OFFSETS, with their undistorted position at TS."""
    cp = cp_4k(suppress)
    gx, gy = np.meshgrid(np.linspace(0.0, W4K, 385), np.linspace(0.0, H4K, 217))
    pts = np.c_[gx.ravel(), gy.ravel()].astype(F32)
    ok = np.ones(len(pts), bool)
    for off in np.r_[OFFSETS, 0.0]:
        for ts in (TS, NTS):
            t = ts / 1000.0 - off
            u = oracle_points(cp, LENS4K, None, pts, t, np_sync.frame_at_timestamp(t, FPS), 1.0, False)
            ok &= (u[:, 0] > 8) & (u[:, 0] < W4K - 8) & (u[:, 1] > 8) & (u[:, 1] < H4K - 8)
    return pts[ok], oracle_points(cp, LENS4K, None, pts[ok], TS / 1000.0, np_sync.frame_at_timestamp(TS / 1000.0, FPS), 1.0, False)


def realistic_pair(n, seed, suppress, tie_at=None):
    """n matched points of a 4K fisheye clip: 80 % moved by a small flow plus noise, 10 % wrong matches between far apart points of the
    visible frame (hundreds to thousands of px long, some from corner to corner, over 4096 px), 10 % copies of one small-flow match.
    tie_at: (small, tied, far) instead — `small` small-flow matches, `tied` copies of one wrong match (corner to corner when `far`,
    else about 400 px long), the rest wrong matches."""
    rng = np.random.default_rng(seed)
    pool, up = _visible_pool(suppress)
    if tie_at is None:
        n_small, n_wrong = int(n * 0.8), n // 10
        n_tie = n - n_small - n_wrong
    else:
        n_small, n_tie, far = tie_at
        n_wrong = n - n_small - n_tie
    # small flow: points well inside, moved by (3.5, -2) px plus noise
    inner = pool[(up[:, 0] > 200) & (up[:, 0] < W4K - 200) & (up[:, 1] > 200) & (up[:, 1] < H4K - 200)]
    a = inner[rng.integers(0, len(inner), n_small)] + rng.random((n_small, 2)).astype(F32)
    small = (a, a + F32([3.5, -2.0]) + rng.normal(0, 0.7, (n_small, 2)).astype(F32))
    # wrong matches: half between random visible points, half between opposite corners of the visible frame
    s = up.sum(axis=1)
    lo, hi = pool[np.argsort(s)[:40]], pool[np.argsort(s)[-40:]]
    n_far = n_wrong // 2
    w1 = np.r_[pool[rng.integers(0, len(pool), n_wrong - n_far)], lo[rng.integers(0, 40, n_far)]]
    w2 = np.r_[pool[rng.integers(0, len(pool), n_wrong - n_far)], hi[rng.integers(0, 40, n_far)]]
    # the tie: one match repeated; a small-flow one, or with tie_at a wrong one
    if tie_at is None:
        t1, t2 = small[0][:1], small[1][:1]
    else:
        t1, t2 = (lo[:1], hi[-1:]) if far else (small[0][:1], small[0][:1] + F32([400.0, 0.0]))
    p1 = np.r_[small[0], w1, np.repeat(t1, n_tie, axis=0)].astype(F32)
    p2 = np.r_[small[1], w2, np.repeat(t2, n_tie, axis=0)].astype(F32)
    perm = rng.permutation(n)
    return (TS, p1[perm]), (NTS, p2[perm])


def realistic_pairs(suppress):
    """The lists for a 4K fisheye clip with the rotation on or suppressed (their wrong matches reach the edges of what is visible)."""
    return [realistic_pair(700, 1, suppress), realistic_pair(1000, 2, suppress, tie_at=(600, 350, True)),
            realistic_pair(2000, 3, suppress, tie_at=(1500, 450, False)), realistic_pair(9000, 4, suppress)]


W_MAX = 32768                         # the largest frame; opencv_standard without distortion and no rotation maps every point to itself
MAX_POINTS = (2 ** 53 - 1) // (2 * W_MAX * W_MAX)      # the largest sum(n) sync_check accepts on a 32768 x 32768 frame


def cp_max():
    cp = make_cp(w=W_MAX, h=W_MAX, lens="opencv_standard")
    cp.c.distortion_coeffs[:] = [0.0] * 12
    cp.c.suppress_rotation = 1
    return cp


def corner_pair(n, seed):
    """n points near one corner of the 32768 frame matched to points near the opposite one, every direction: keys just below 2^31,
    two matches from the smallest undistorted coordinate above 0 to the largest below 32768 (key 2^31 - 512) and one from 0
    (outside)."""
    rng = np.random.default_rng(seed)
    near = rng.random((n, 2)) * 48.0
    sx, sy = rng.integers(0, 2, n), rng.integers(0, 2, n)
    a = np.c_[np.where(sx, near[:, 0], W_MAX - near[:, 0]), np.where(sy, near[:, 1], W_MAX - near[:, 1])]
    b = np.c_[np.where(sx, W_MAX - near[:, 1], near[:, 1]), np.where(sy, W_MAX - near[:, 0], near[:, 0])]
    a, b = a.astype(F32), b.astype(F32)
    top = np.nextafter(F32(W_MAX), F32(0))
    tiny = F32(1e-3)                                     # 2^-10 undistorted; the smallest float above 0 comes out as 0
    a[:3] = [[tiny, tiny], [top, tiny], [0.0, 5.0]]
    b[:3] = [[top, top], [tiny, top], [W_MAX - 5.0, W_MAX - 5.0]]
    return (TS, a), (NTS, b)


def _sized(n, seed, suppress):
    """A pair of n points: realistic_pair, cut down below 10 points, empty for 0."""
    if n == 0:
        return (TS, np.zeros((0, 2), F32)), (NTS, np.zeros((0, 2), F32))
    if n < 10:
        (ts, p1), (nts, p2) = realistic_pair(10, seed, suppress)
        return (ts, p1[:n]), (nts, p2[:n])
    return realistic_pair(n, seed, suppress)


# ---- the inside test's edges ----------------------------------------------------------------------------------------------------------
def _ulp_range(a, b, extra=8):
    """Every float32 from `extra` ulps below min(a, b) to `extra` above max(a, b)."""
    lo, hi = F32(min(a, b)), F32(max(a, b))
    for _ in range(extra):
        lo, hi = np.nextafter(lo, F32(-np.inf)), np.nextafter(hi, F32(np.inf))
    ia, ib = np.array([lo, hi], F32).view(np.int32)
    assert lo > 0 and ib - ia < 1_000_000
    return np.arange(ia, ib + 1, dtype=np.int32).view(F32)


def edge_inputs(points, axis, fixed, lo, hi, target):
    """Inputs along one line (coordinate `axis` varies over [lo, hi], the other is `fixed`) whose undistorted coordinate `axis` equals
    `target`, found by bisection and then a float-step search.  Returns (inputs (m, 2), their outputs, exact): the inputs landing on
    `target` when some do, else the two adjacent floats whose outputs bracket it.  The output is increasing along the line."""
    def at(vals):
        pts = np.zeros((len(vals), 2), F32)
        pts[:, axis], pts[:, 1 - axis] = vals, fixed
        return pts, points(pts)[:, axis]
    t = F32(target)
    for _ in range(8):
        vals = np.linspace(lo, hi, 1025).astype(F32)
        _, out = at(vals)
        i = int(np.searchsorted(out, t))           # first output >= target
        assert 0 < i < len(vals), (axis, target, out[0], out[-1])
        lo, hi = float(vals[i - 1]), float(vals[i])
        if np.nextafter(F32(lo), F32(np.inf)) >= F32(hi):
            break
    vals = _ulp_range(lo, hi)
    pts, out = at(vals)
    hit = out == t
    if hit.any():
        return pts[hit], out[hit], True
    j = int(np.flatnonzero((out[:-1] < t) & (out[1:] > t))[0])
    return pts[j:j + 2], out[j:j + 2], False


def edge_pairs(points, w, h, cx, cy):
    """Point pairs on the inside test's edges: for each coordinate, inputs whose undistorted coordinate is exactly 0, the smallest float
    above 0, the largest float below the frame size and exactly the frame size (or the two inputs that bracket each), searched along
    the lines through (cx, cy).  Each edge input is matched with a point moved 3 px inwards, as the first and as the second point of a
    pair, next to 40 small-flow matches well inside."""
    targets = []
    for axis, size, fixed in ((0, w, cy), (1, h, cx)):
        for tgt, lo, hi in ((0.0, 1.0, cx if axis == 0 else cy), (float(np.nextafter(F32(0), F32(1))), 1.0, cx if axis == 0 else cy),
                            (float(np.nextafter(F32(size), F32(0))), cx if axis == 0 else cy, size - 1.0), (float(size), cx if axis == 0 else cy, size - 1.0)):
            pts, out, exact = edge_inputs(lambda p: points(p), axis, fixed, lo, hi, tgt)
            targets.append((axis, tgt, pts, out, exact))
    e = np.concatenate([t[2] for t in targets]).astype(F32)
    inward = np.sign(F32([cx, cy]) - e).astype(F32) * F32(3.0)
    rng = np.random.default_rng(77)
    fill = (np.array([cx, cy], F32) + (rng.random((40, 2)) - 0.5).astype(F32) * F32([0.5 * w, 0.5 * h])).astype(F32)
    p1 = np.r_[e, e + inward, fill].astype(F32)
    p2 = np.r_[e + inward, e, fill + F32([2.0, 1.0])].astype(F32)
    return [((TS, p1), (NTS, p2))], targets


# ---- without a GPU: the lists do what the GPU tests need --------------------------------------------------------------------------------
def test_reference_on_small_cases():
    """The integer reference itself: k = int(m * 0.9) with 0.9 in f64, NO_KEY never counts."""
    assert [k_of(m) for m in (0, 1, 2, 9, 10, 11, 19, 20, 1000, MAX_POINTS)] == [0, 0, 1, 8, 9, 9, 17, 18, 900, int(MAX_POINTS * 0.9)]
    assert select_sum([5, NO_KEY, 3, 9, 1, NO_KEY, 7, 2, 8, 6, 4, 0]) == sum(range(9))
    assert select_sum([NO_KEY, 7]) == 0 and select_sum([]) == 0
    assert kth([4, 4, 4, 1, 9, 4, 4, 4, 4, 4]) == (9, 4, 1, 8)


def test_realistic_lists_reach_every_pass_and_tie_across_k():
    """The 4K fisheye lists, rotation suppressed and on, through the oracle: keys of at least 2^24 (pass 1 sees non-zero bytes), keys
    between 2^16 and 2^24, the copied matches tie, and in the tie lists the tie starts below the k-th key and ends above it, once with
    the k-th key at or above 2^24.  The oracle's cost equals the integer reference on keys from its own points."""
    for suppress in (True, False):
        pairs = realistic_pairs(suppress)
        cp = cp_4k(suppress)
        pts = oracle_pts(cp, LENS4K)
        for off in (0.0, 7.25):
            keys = [pair_keys(pts, p, off, W4K, H4K) for p in pairs]
            valid = np.concatenate([k[k != NO_KEY] for k in keys])
            assert (valid >= 2 ** 24).sum() >= 20 and ((valid >= 2 ** 16) & (valid < 2 ** 24)).sum() >= 50, suppress
            assert all((k == NO_KEY).sum() < k.size // 20 for k in keys)
            for i, k in enumerate(keys):
                kk, t, below, eq = kth(k)
                vals, counts = np.unique(k[k != NO_KEY], return_counts=True)
                assert counts.max() >= len(k) // 12, (i, counts.max())          # the copied match ties
                if i in (1, 2):
                    assert below < kk < below + eq, (i, kk, below, eq)          # the tie spans the k-th key
                    assert (t >= 2 ** 24) == (i == 1), (i, t)
            want = np.array([float(sum(select_sum(pair_keys(pts, p, off, W4K, H4K)) for p in pairs))])
            assert same(oracle_costs(cp, LENS4K, None, pairs, [off]), want), suppress


def test_max_frame_and_2_53_lists():
    """On the 32768 x 32768 frame every point is its own undistorted point: the corner pairs give keys just below 2^31, down
    to 2^31 - 512, the match from 0 none; the job of MAX_POINTS such points stays one point under the 2^53 bound and its sum of keys
    is above 0.8 * 2^53.  Both costs equal the oracle's."""
    cp = cp_max()
    pts = oracle_pts(cp, "opencv_standard")
    small = [corner_pair(3000, 21)]
    k = pair_keys(pts, small[0], 0.0, W_MAX, W_MAX)
    assert k[0] == k[1] == 2 ** 31 - 512 and k[2] == NO_KEY and (k[3:] > 2 ** 31 - 2 ** 24).all(), k[:4]
    assert same(oracle_costs(cp, "opencv_standard", None, small, [0.0]), [float(select_sum(k))])
    assert MAX_POINTS * 2 * W_MAX ** 2 < 2 ** 53 <= (MAX_POINTS + 1) * 2 * W_MAX ** 2
    job = _max_job()
    keys = np.concatenate([pair_keys(pts, p, 0.0, W_MAX, W_MAX) for p in job])
    assert keys.size == MAX_POINTS
    total = sum(select_sum(pair_keys(pts, p, 0.0, W_MAX, W_MAX)) for p in job)
    assert 0.8 * 2 ** 53 < total < 2 ** 53
    assert same(oracle_costs(cp, "opencv_standard", None, job, [0.0]), [float(total)])


def _max_job():
    """MAX_POINTS points in one big pair and one of 1000 (sum(n) one below the 2^53 refusal)."""
    (ts, a), (nts, b) = corner_pair(MAX_POINTS - 1000, 22)
    return [((ts, a), (nts, b)), corner_pair(1000, 23)]


def test_edge_search_finds_the_edges():
    """The float-step search through the oracle's point path (rotation suppressed: the device's equals it bit for bit) finds, for each
    edge of the inside test, an input landing on it or two adjacent inputs bracketing it; the edge pairs include keys on both sides."""
    cp = cp_4k(True)
    pts = oracle_pts(cp, LENS4K)
    pairs, targets = edge_pairs(lambda p: pts(p, TS / 1000.0, 1), W4K, H4K, W4K / 2.0, H4K / 2.0)
    for axis, tgt, p, out, exact in targets:
        t = F32(tgt)
        assert (exact and (out == t).all()) or (not exact and out[0] < t < out[1]), (axis, tgt, out)
        assert abs(float(out[0]) - tgt) < 1e-2
    k = pair_keys(pts, pairs[0], 0.0, W4K, H4K)
    assert (k == NO_KEY).sum() >= 8 and (k[:-40] != NO_KEY).sum() >= 8, k
    assert same(oracle_costs(cp, LENS4K, None, pairs, OFFSETS), exact_costs(pts, pairs, OFFSETS, W4K, H4K))


# ---- raw keys on the device ------------------------------------------------------------------------------------------------------------
def _raw_cases():
    """(name, keys) groups: every case of the selection the point path could send it, and some it cannot (keys above 2^31)."""
    rng = np.random.default_rng(2024)
    cases = []
    for v in (0, 255, 256, 65535, 65536, 2 ** 24 - 1, 2 ** 24, 2 ** 31 - 1, 2 ** 31, NO_KEY - 1):
        cases.append(("equal %d" % v, np.full(1000, v, np.uint32)))
    # the k-th key inside a tie that starts below it and ends above it, at each byte
    for t in (77, 0x1234, 0x56789A, 0x3456789A):
        keys = np.r_[rng.integers(0, t, 600), np.full(350, t), rng.integers(t + 1, 2 ** 31, 50)]
        cases.append(("tie at %#x" % t, rng.permutation(keys).astype(np.uint32)))
    cases.append(("byte 3 only", ((rng.integers(0, 128, 3000) << 24) | 0x00A5A5A5).astype(np.uint32)))
    cases.append(("byte 0 only", (0x12345600 | rng.integers(0, 256, 3000)).astype(np.uint32)))
    cases.append(("byte 3 only, with ties", ((rng.integers(0, 4, 3000) << 24) | 0x00FFFFFF).astype(np.uint32)))
    # the k-th key in bin 0 and in bin 255 of each pass, its prefix shared with keys on both sides
    for shift in (24, 16, 8, 0):
        for b in (0, 255):
            high = (0x5A3C7E00 >> (shift + 8) << (shift + 8)) if shift < 24 else 0
            low = (1 << shift) // 2
            t = high | (b << shift) | low
            n = 2000
            k = k_of(n)
            span = 1 << (shift + 9) if shift < 24 else 1 << 30
            below = rng.integers(max(0, t - span), t, k - 1)
            above = rng.integers(t + 1, min(NO_KEY, t + span), n - k)
            cases.append(("bin %d of pass %d" % (b, (24 - shift) // 8 + 1), rng.permutation(np.r_[below, [t], above]).astype(np.uint32)))
    for frac in (0.1, 0.12):                           # 10 % and 12 % outliers above 2^24
        n = 5000; no = int(n * frac)
        keys = np.r_[rng.integers(0, 5000, n - no), rng.integers(2 ** 24, 2 ** 31 + 1, no)]
        cases.append(("outliers %.2f" % frac, rng.permutation(keys).astype(np.uint32)))
    for m, n in ((0, 300), (1, 300), (2, 300), (10, 300), (10, 10), (1, 1), (300, 300), (9000, 9000), (10, 9000)):
        keys = np.full(n, NO_KEY, np.uint32)
        at = np.sort(rng.choice(n, m, replace=False))
        keys[at] = rng.integers(0, 2 ** 20, m)
        cases.append(("m=%d of n=%d" % (m, n), keys))
    for n in (1, 255, 256, 257, 511, 513, SMEM_KEYS - 1, SMEM_KEYS, SMEM_KEYS + 1, 20_000):
        keys = rng.integers(0, 2 ** 31 + 1, n).astype(np.uint32)
        keys[rng.random(n) < 0.05] = NO_KEY
        cases.append(("n=%d" % n, keys))
    for seed in range(6):
        r = np.random.default_rng(seed)
        n = int(r.integers(1000, 30_000))
        keys = r.integers(0, 2 ** 31, n).astype(np.uint32)
        keys[r.random(n) < 0.03] = NO_KEY
        cases.append(("random seed %d" % seed, keys))
    return cases


def test_raw_cases_are_what_they_say():
    """The raw-key cases really put the k-th key where their names say (no GPU needed)."""
    for name, keys in _raw_cases():
        k, t, below, eq = kth(keys)
        if name.startswith("tie"):
            assert below < k < below + eq, name
        if name.startswith("bin"):
            b, p = int(name.split()[1]), int(name.split()[-1])
            shift = 24 - 8 * (p - 1)
            assert (t >> shift) & 255 == b and eq == 1, name
            pref = [x for x in keys if (x >> (shift + 8)) == (t >> (shift + 8))] if shift < 24 else keys
            assert len({(x >> shift) & 255 for x in pref}) > 2, name              # the pass sees other bins too
        if name.startswith("outliers"):
            assert (np.asarray(keys) >= 2 ** 24).sum() >= len(keys) // 10
        if name.startswith("m="):
            assert int((keys != NO_KEY).sum()) == int(name[2:].split()[0])


@pytest.mark.gpu
def test_raw_keys_match_integer_reference():
    """gf_cuda_selftest_sync_select on every raw-key case, all in one launch and each on its own, equals the sorted integer sum."""
    cases = _raw_cases()
    want = np.array([select_sum(k) for _, k in cases], np.uint64)
    got = g.selftest_sync_select([k for _, k in cases])
    bad = [(cases[i][0], int(got[i]), int(want[i])) for i in np.flatnonzero(got != want)]
    assert not bad, bad
    for (name, keys), w in zip(cases, want):
        assert int(g.selftest_sync_select([keys])[0]) == int(w), name
    assert g.selftest_sync_select([]).size == 0


# ---- end to end on the device ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_realistic_lists_end_to_end():
    """The 4K fisheye lists: with the rotation on, costs equal the integer reference on keys from gf_cuda_undistort_points; with it
    suppressed, they equal the reference and the oracle, and find_sync_offsets equals the oracle's search."""
    for suppress in (False, True):
        pairs = realistic_pairs(suppress)
        cp = cp_4k(suppress)
        dg = g.DeviceGyro(cp)
        try:
            got = dg.sync_costs(LENS4K, None, FPS, pairs, offsets_ms=OFFSETS)
            assert same(got, exact_costs(device_pts(dg, LENS4K), pairs, OFFSETS, W4K, H4K)), (suppress, got)
            if suppress:
                assert same(got, oracle_costs(cp, LENS4K, None, pairs, OFFSETS)), got
                ranges = [(0, 100_000, pairs)]
                dev = dg.find_sync_offsets(LENS4K, None, FPS, ranges, 0.0, 40.0)
                ora = oracle_find(cp, LENS4K, None, ranges, 0.0, 40.0, False)
                assert dev == ora and all(same(a, b) for a, b in zip(dev, ora)), (dev, ora)
        finally:
            dg.close()


@pytest.mark.gpu
def test_inside_test_edges():
    """Pairs on the inside test's edges, found by the float-step search through gf_cuda_undistort_points: costs equal the reference on
    the device's points and the oracle (rotation suppressed)."""
    cp = cp_4k(True)
    dg = g.DeviceGyro(cp)
    try:
        pts = device_pts(dg, LENS4K)
        pairs, targets = edge_pairs(lambda p: pts(p, TS / 1000.0, 1), W4K, H4K, W4K / 2.0, H4K / 2.0)
        for axis, tgt, p, out, exact in targets:
            assert (exact and (out == F32(tgt)).all()) or (not exact and out[0] < F32(tgt) < out[1]), (axis, tgt, out)
        got = dg.sync_costs(LENS4K, None, FPS, pairs, offsets_ms=OFFSETS)
        assert same(got, exact_costs(pts, pairs, OFFSETS, W4K, H4K)), got
        assert same(got, oracle_costs(cp, LENS4K, None, pairs, OFFSETS)), got
    finally:
        dg.close()


@pytest.mark.gpu
def test_max_frame_and_job_just_under_2_53():
    """Keys just below 2^31 on a 32768 x 32768 frame, and a job of MAX_POINTS points whose cost is above 0.8 * 2^53: exact
    against the reference and the oracle; one more point is refused."""
    cp = cp_max()
    dg = g.DeviceGyro(cp)
    try:
        pts = device_pts(dg, "opencv_standard")
        small = [corner_pair(3000, 21)]
        got = dg.sync_costs("opencv_standard", None, FPS, small, offsets_ms=[0.0, 5.0])
        assert same(got, exact_costs(pts, small, [0.0, 5.0], W_MAX, W_MAX)), got
        job = _max_job()
        got = dg.sync_costs("opencv_standard", None, FPS, job, offsets_ms=[0.0])
        want = oracle_costs(cp, "opencv_standard", None, job, [0.0])
        assert same(got, want) and got[0] > 0.8 * 2 ** 53, (got, want)
        assert same(got, exact_costs(pts, job, [0.0], W_MAX, W_MAX)), got
        (ts, a), (nts, b) = job[1]
        over = job[:1] + [((ts, np.r_[a, a[:1]]), (nts, np.r_[b, b[:1]]))]
        with pytest.raises(g.GyroflowCoreError) as e:
            dg.sync_costs("opencv_standard", None, FPS, over, offsets_ms=[0.0])
        assert "2^53" in str(e.value)
    finally:
        dg.close()


@pytest.mark.gpu
def test_mixed_launch():
    """One launch with empty, shared-memory and global-scratch pairs (0, 1, 5, 300, 8192, 8193 and 20000 points): exact against the
    reference (rotation on and suppressed) and the oracle (suppressed)."""
    for suppress in (False, True):
        pairs = [_sized(n, 10 + i, suppress) for i, n in enumerate([0, 5, 300, SMEM_KEYS, 0, SMEM_KEYS + 1, 20_000, 1])]
        cp = cp_4k(suppress)
        dg = g.DeviceGyro(cp)
        try:
            got = dg.sync_costs(LENS4K, None, FPS, pairs, offsets_ms=OFFSETS)
            assert same(got, exact_costs(device_pts(dg, LENS4K), pairs, OFFSETS, W4K, H4K)), (suppress, got)
            if suppress:
                assert same(got, oracle_costs(cp, LENS4K, None, pairs, OFFSETS)), got
        finally:
            dg.close()


def _chunk_size(dg, pairs):
    """The candidates per chunk of a search over `pairs`: the largest n whose sync_costs call takes one chunk."""
    chunks = lambda n: (dg.sync_costs(LENS4K, None, FPS, pairs, offsets_ms=np.zeros(n)), dg.sync_timing()["chunks"])[1]
    lo, hi = 1, 2
    while chunks(hi) == 1:
        lo, hi = hi, 2 * hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if chunks(mid) == 1 else (lo, mid)
    return lo


@pytest.mark.gpu
def test_big_pair_over_three_chunks():
    """A 9000-point pair (global scratch) next to 600 two-point pairs and an empty one, over 2 * chunk + 1 candidates: three chunks, the
    last with a single candidate.  With the rotation on every candidate's cost differs and equals the reference on the device's
    points; with it suppressed the costs and the search equal the oracle."""
    rng = np.random.default_rng(5)
    big = realistic_pair(9000, 31, False)
    (_, a), (_, b) = realistic_pair(1200, 32, False)
    pairs = [big] + [((TS, a[2 * i:2 * i + 2]), (NTS, b[2 * i:2 * i + 2])) for i in range(600)] + [_sized(0, 0, False)]
    cp = cp_4k(False)
    dg = g.DeviceGyro(cp)
    try:
        chunk = _chunk_size(dg, pairs)
        assert 2 <= chunk <= 200, chunk
        offsets = np.sort(rng.uniform(-30.0, 30.0, 2 * chunk + 1))
        got = dg.sync_costs(LENS4K, None, FPS, pairs, offsets_ms=offsets)
        assert dg.sync_timing()["chunks"] == 3
        assert len(set(got)) > 0.9 * len(got)
        assert same(got, exact_costs(device_pts(dg, LENS4K), pairs, offsets, W4K, H4K)), got
        s1, s2 = _streams()
        assert same(dg.sync_costs(LENS4K, None, FPS, pairs, offsets_ms=offsets, stream=s1.cuda_stream), got)
        assert same(dg.sync_costs(LENS4K, None, FPS, pairs, offsets_ms=offsets, stream=s2.cuda_stream), got)
    finally:
        dg.close()
    cp = cp_4k(True)
    dg = g.DeviceGyro(cp)
    try:
        offsets = np.linspace(-40.0, 40.0, 2 * chunk + 1)          # the records take the IBIS data of frames 0 .. 2
        got = dg.sync_costs(LENS4K, None, FPS, pairs, offsets_ms=offsets)
        assert dg.sync_timing()["chunks"] == 3
        assert same(got, oracle_costs(cp, LENS4K, None, pairs, offsets)), got
        ranges = [(0, 100_000, pairs)]
        dev = dg.find_sync_offsets(LENS4K, None, FPS, ranges, 0.0, float(2 * chunk + 1))
        ora = oracle_find(cp, LENS4K, None, ranges, 0.0, float(2 * chunk + 1), False)
        assert dev == ora and all(same(x, y) for x, y in zip(dev, ora)), (dev, ora)
    finally:
        dg.close()


def _streams():
    import torch
    return torch.cuda.Stream(), torch.cuda.Stream()


@pytest.mark.gpu
def test_two_streams_give_identical_costs():
    """The realistic lists with the rotation on, on two torch streams in turn and on the gyro object's own stream: identical costs."""
    pairs = realistic_pairs(False)
    dg = g.DeviceGyro(cp_4k(False))
    try:
        s1, s2 = _streams()
        a = dg.sync_costs(LENS4K, None, FPS, pairs, offsets_ms=OFFSETS, stream=s1.cuda_stream)
        b = dg.sync_costs(LENS4K, None, FPS, pairs, offsets_ms=OFFSETS, stream=s2.cuda_stream)
        c = dg.sync_costs(LENS4K, None, FPS, pairs, offsets_ms=OFFSETS)
        assert same(a, b) and same(a, c), (a, b, c)
    finally:
        dg.close()
