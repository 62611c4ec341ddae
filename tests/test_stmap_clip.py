"""ST maps of a whole clip (SURVEY f4): gf_cuda_stmap_sizes + gf_cuda_generate_stmaps_dev against the single-frame
gf_cuda_generate_stmap, frame by frame and bit for bit, and one frame per option row against the oracle (generate_stmaps,
src/core/stmap.rs:6-146)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi
from tests.test_kernel_matrix import REFERENCE_PAIRS
from tests.test_point_matrix import LENS_A, LENS_B, POINT_PAIRS, STMAP_SIZE, _scaled, first_diff, same_bits
from tests.test_stmap import oracle_stmap
from tests.test_zoom import _distorting_mesh, _zoom_stab, make_cp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GF_OK, GF_ERR_BAD_PARAMS, GF_ERR_SIZE_MISMATCH, GF_ERR_UNSUPPORTED_COMBO, GF_ERR_BUFFER_TOO_SMALL = 0, -1, -3, -5, -7
SENTINEL = 0x7FA5A5A5                  # a NaN no kernel writes
# a clip of five frames with distinct timestamps, not in frame order
CLIP_FRAMES = [0, 1, 2, 3, 4]
CLIP_TS = [300.0, 1234.5, 700.0, 2100.0, 2900.0]
ORACLE_ENTRY = 2                       # the frame of each row that is also compared with the oracle


def test_new_symbols_are_declared_and_exported():
    """The clip entry points are in the header's ST-map block, in the ctypes mirror and exported by the library."""
    lib = g.load_library()
    header = open(os.path.join(ROOT, "include", "gyroflow_cuda.h")).read()
    declared = set(re.findall(r"GF_API\s+[\w\s\*]+?\b(gf_\w+)\s*\(", header))
    bound = {n for n, _, _ in abi.EXPORTS}
    for name in ("gf_cuda_stmap_sizes", "gf_cuda_generate_stmaps_dev"):
        assert name in declared and name in bound and hasattr(lib, name), name
    assert header.index("gf_cuda_generate_stmap(") < header.index("gf_cuda_stmap_sizes(") < header.index("gf_cuda_generate_stmaps_dev(")


# ---- option rows: (name, per_frame, make_cp arguments for a w x h frame, oracle cp of one frame or None for the clip's own) ---------------
def _lens_frames(w, h):
    return [_scaled(LENS_A if i % 2 == 0 else LENS_B, w, h) for i in range(len(CLIP_FRAMES))]


def _meshes(w, h):
    return [_distorting_mesh(w, h, False, 9), None, _distorting_mesh(w, h, True, 9), _distorting_mesh(w, h, True, 7), None]


ROWS = [
    ("per-frame", True, lambda w, h: {}),
    ("not-per-frame", False, lambda w, h: {}),
    ("horizontal", True, lambda w, h: dict(horizontal=True)),
    ("ibis-rs", True, lambda w, h: dict(camera_stab=_zoom_stab(5, h))),
    ("ibis-not-per-frame", False, lambda w, h: dict(camera_stab=_zoom_stab(5, h))),
    ("mesh", True, lambda w, h: dict(distorting_meshes=_meshes(w, h), camera_stab=_zoom_stab(5, h))),
    ("lens-per-frame", True, lambda w, h: dict(lens_per_frame=_lens_frames(w, h))),
]


def row_cp(kw, lens, digital, w, h):
    cp = make_cp(w=w, h=h, lens=lens, digital=digital, **kw(w, h))
    return cp


def oracle_cp(name, kw, lens, digital, w, h, frame):
    """The oracle takes no per-frame lens: for that row it gets a ComputeParams whose constants are the frame's lens."""
    if name != "lens-per-frame":
        return row_cp(kw, lens, digital, w, h)
    cp = make_cp(w=w, h=h, lens=lens, digital=digital)
    L = _lens_frames(w, h)[frame]
    cp.c.camera_matrix[:] = L["camera_matrix"]; cp.c.distortion_coeffs[:] = L["distortion_coeffs"]
    return cp


def single_sizes(dg, lens, digital, per_frame):
    """Each frame's size query of gf_cuda_generate_stmap: [(rc, new_w, new_h)]."""
    m, d = abi.LENS[lens], abi.LENS[digital] if digital else 0
    out = []
    for frame, ts in zip(CLIP_FRAMES, CLIP_TS):
        nw, nh = C.c_int32(), C.c_int32()
        rc = dg._lib.gf_cuda_generate_stmap(dg._h, C.byref(dg.cp.c), m, d, int(per_frame), frame, ts, C.byref(nw), C.byref(nh), None, 0, None, 0, None)
        out.append((rc, nw.value, nh.value))
    return out


def clip_sizes(dg, lens, digital, per_frame, frames=CLIP_FRAMES, ts=CLIP_TS):
    """gf_cuda_stmap_sizes straight through the C ABI: (rc, new_w[], new_h[]), the arrays as written even when the call fails."""
    fr = np.asarray(frames, np.uintp); t = np.asarray(ts, np.float64)
    nw, nh = np.full(fr.size, -7, np.int32), np.full(fr.size, -7, np.int32)
    rc = dg._lib.gf_cuda_stmap_sizes(dg._h, C.byref(dg.cp.c), abi.LENS[lens], abi.LENS[digital] if digital else 0, int(per_frame),
                                     fr.ctypes.data, t.ctypes.data, fr.size, nw.ctypes.data, nh.ctypes.data, None)
    return rc, nw, nh


@pytest.mark.gpu
@pytest.mark.parametrize("lens,digital", POINT_PAIRS, ids=["%s+%s" % (l, d) for l, d in POINT_PAIRS])
def test_clip_matches_single_frame_and_oracle(lens, digital):
    """Every option row on a STMAP_SIZE frame: the clip's sizes are the single-frame call's, both maps of every frame are byte-identical
    to the single-frame call's, and one frame per row is byte-identical to the oracle.  The single-frame calls share the gyro's warp
    context with the clip: the smallest frame's call before the clip starts it at that frame's size, the clip reuses or replaces it, and
    each call after the clip reuses the clip's context set to its frame's size."""
    sw, sh = STMAP_SIZE
    bad, compared = [], 0
    for name, per_frame, kw in ROWS:
        dg = g.DeviceGyro(row_cp(kw, lens, digital, sw, sh))
        try:
            want_sizes = single_sizes(dg, lens, digital, per_frame)
            rc, nw, nh = clip_sizes(dg, lens, digital, per_frame)
            if [(w, h) for _, w, h in want_sizes] != list(zip(nw.tolist(), nh.tolist())):
                bad.append("%s: sizes %s != single-frame %s" % (name, list(zip(nw, nh)), want_sizes))
                continue
            single_rc = next((r for r, _, _ in want_sizes if r != GF_OK), GF_OK)
            if rc != single_rc:
                bad.append("%s: gf_cuda_stmap_sizes returned %d, the single-frame size query %d" % (name, rc, single_rc))
                continue
            if rc != GF_OK:                                    # an undistorted size out of range: nothing to render
                continue
            if (lens, digital) not in REFERENCE_PAIRS:         # the warp renders the undistort map and has no kernel for this pair
                with pytest.raises(g.GyroflowCoreError) as e:
                    dg.generate_stmaps(lens, digital, CLIP_TS, CLIP_FRAMES, per_frame)
                assert e.value.code == GF_ERR_UNSUPPORTED_COMBO
                continue
            small = int(np.argmin(nw.astype(np.int64) * nh))
            before = dg.generate_stmap(lens, digital, CLIP_TS[small], CLIP_FRAMES[small], per_frame)
            dists, undists = dg.generate_stmaps(lens, digital, CLIP_TS, CLIP_FRAMES, per_frame)
            dists = [t.cpu().numpy() for t in dists]; undists = [t.cpu().numpy() for t in undists]
            singles = [(small, "before the clip", before)]
            singles += [(i, "after the clip", dg.generate_stmap(lens, digital, ts, frame, per_frame)) for i, (frame, ts) in enumerate(zip(CLIP_FRAMES, CLIP_TS))]
            for i, when, (want_dist, want_und) in singles:
                for what, got, want in (("redistort", dists[i], want_dist), ("undistort", undists[i], want_und)):
                    compared += 1
                    if not same_bits(got, want).all():
                        bad.append("%s frame %d %s map vs single frame %s: %s" % (name, CLIP_FRAMES[i], what, when, first_diff(got, want)))
            frame, ts = CLIP_FRAMES[ORACLE_ENTRY], CLIP_TS[ORACLE_ENTRY]
            onw, onh, o_dist, o_und = oracle_stmap(oracle_cp(name, kw, lens, digital, sw, sh, frame), lens, digital, ts, frame, per_frame)
            if o_dist is None or (onw, onh) != (nw[ORACLE_ENTRY], nh[ORACLE_ENTRY]):
                bad.append("%s frame %d: oracle size %dx%d, clip %dx%d" % (name, frame, onw, onh, nw[ORACLE_ENTRY], nh[ORACLE_ENTRY]))
                continue
            for what, got, want in (("redistort", dists[ORACLE_ENTRY], o_dist), ("undistort", undists[ORACLE_ENTRY], o_und)):
                compared += 1
                if not same_bits(got, want).all():
                    bad.append("%s frame %d %s map vs oracle: %s" % (name, frame, what, first_diff(got, want)))
        finally:
            dg.close()
    assert not bad, bad
    assert compared > 0 or (lens, digital) not in REFERENCE_PAIRS


def _checksums(lib, maps, stream):
    """One device checksum per map, enqueued on `stream` (gf_cuda_checksum_dev)."""
    import torch
    out = torch.zeros(len(maps), dtype=torch.int64, device="cuda")
    for i, t in enumerate(maps):
        assert lib.gf_cuda_checksum_dev(t.data_ptr(), t.numel() * 4, out.data_ptr() + 8 * i, stream) == 0
    return out


@pytest.mark.gpu
def test_job_on_a_caller_stream_is_ordered_without_synchronisation():
    """The job and a device-side checksum of its outputs on a side stream, nothing synchronised in between: the checksums and the maps
    equal those of the same job run synchronously."""
    import torch
    w, h = 640, 360
    cp = make_cp(w=w, h=h, camera_stab=_zoom_stab(8, h))
    ts, frames = [100.0 + 97.0 * i for i in range(8)], list(range(8))
    dg = g.DeviceGyro(cp)
    try:
        want_d, want_u = dg.generate_stmaps("opencv_fisheye", None, ts, frames, True)
        torch.cuda.synchronize()
        want_sum = _checksums(dg._lib, want_d + want_u, None).cpu()
        want_d = [t.cpu() for t in want_d]; want_u = [t.cpu() for t in want_u]
        side = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            got_d, got_u = dg.generate_stmaps("opencv_fisheye", None, ts, frames, True, stream=side.cuda_stream)
            got_sum = _checksums(dg._lib, got_d + got_u, side.cuda_stream)
            got_sum_host = got_sum.to("cpu", non_blocking=True)
        side.synchronize()
        assert torch.equal(got_sum_host, want_sum)
        for a, b in zip(got_d + got_u, want_d + want_u):
            assert torch.equal(a.cpu().view(torch.int32), b.view(torch.int32))
    finally:
        dg.close()


@pytest.mark.gpu
def test_two_jobs_back_to_back_on_one_gyro():
    """Jobs enqueued one after the other without a synchronisation: the second reuses the first one's warp context, the third has
    another lens model and so a new one.  Every map equals the single-frame call's."""
    import torch
    sw, sh = STMAP_SIZE
    fisheye = make_cp(w=sw, h=sh, camera_stab=_zoom_stab(5, sh))
    sony = make_cp(w=sw, h=sh, lens="sony", camera_stab=_zoom_stab(5, sh))       # the same gyro data, the sony lens profile
    dg = g.DeviceGyro(fisheye)
    try:
        jobs = [(fisheye, "opencv_fisheye", None, CLIP_TS, True), (fisheye, "opencv_fisheye", None, CLIP_TS[1:], False),
                (sony, "sony", None, CLIP_TS[::-1], True)]
        results = []
        for cp, lens, dig, ts, pf in jobs:
            dg.cp = cp
            results.append(dg.generate_stmaps(lens, dig, ts, CLIP_FRAMES[:len(ts)], pf))
        torch.cuda.synchronize()
        for (cp, lens, dig, ts, pf), (dists, undists) in zip(jobs, results):
            dg.cp = cp
            for i, t in enumerate(ts):
                want_dist, want_und = dg.generate_stmap(lens, dig, t, CLIP_FRAMES[i], pf)
                assert same_bits(dists[i].cpu().numpy(), want_dist).all(), (lens, i)
                assert same_bits(undists[i].cpu().numpy(), want_und).all(), (lens, i)
    finally:
        dg.close()


@pytest.mark.gpu
def test_single_frame_between_jobs_of_another_lens_pair():
    """A one-frame sony call between two fisheye clip jobs on one gyro, nothing synchronised in between: the one-frame call replaces the
    gyro's warp context while the first job may still use it, and the second job replaces it again.  Every map is byte-identical to the
    same call's on a gyro of its own."""
    import torch
    sw, sh = STMAP_SIZE
    fisheye = make_cp(w=sw, h=sh, camera_stab=_zoom_stab(5, sh))
    sony = make_cp(w=sw, h=sh, lens="sony", camera_stab=_zoom_stab(5, sh))       # the same gyro data, the sony lens profile
    calls = [(fisheye, lambda dg: dg.generate_stmaps("opencv_fisheye", None, CLIP_TS, CLIP_FRAMES, True)),
             (sony, lambda dg: [[m] for m in dg.generate_stmap("sony", None, CLIP_TS[2], CLIP_FRAMES[2], True)]),
             (fisheye, lambda dg: dg.generate_stmaps("opencv_fisheye", None, CLIP_TS[::-1], CLIP_FRAMES, False))]
    shared = g.DeviceGyro(fisheye)
    try:
        got = []
        for cp, call in calls:
            shared.cp = cp
            got.append(call(shared))
        torch.cuda.synchronize()
        for k, (cp, call) in enumerate(calls):
            own = g.DeviceGyro(cp)
            try:
                want = call(own)
                torch.cuda.synchronize()
            finally:
                own.close()
            for maps_got, maps_want in zip(got[k], want):
                assert len(maps_got) == len(maps_want)
                for i, (a, b) in enumerate(zip(maps_got, maps_want)):
                    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
                    b = b.cpu().numpy() if isinstance(b, torch.Tensor) else b
                    assert same_bits(a, b).all(), (k, i, first_diff(a, b))
    finally:
        shared.close()


# ---- errors -----------------------------------------------------------------------------------------------------------------------
class Job:
    """Raw arguments of gf_cuda_generate_stmaps_dev over sentinel-filled device buffers."""

    def __init__(self, dg, n=3, new_w=None, new_h=None, extra=0):
        import torch
        self.dg, self.n = dg, n
        w, h = dg.cp.c.width, dg.cp.c.height
        self.frames = np.arange(n, dtype=np.uintp); self.ts = np.linspace(200.0, 1400.0, n)
        self.nw = np.asarray(new_w if new_w is not None else [w + 4] * n, np.int32)
        self.nh = np.asarray(new_h if new_h is not None else [h + 2] * n, np.int32)
        self.dcap = w * h * 3
        self.ucap = 3 * int((self.nw.astype(np.int64) * self.nh).max()) + extra
        self.bufs = [torch.full((self.dcap,), SENTINEL, dtype=torch.int32, device="cuda") for _ in range(n)]
        self.ubufs = [torch.full((max(self.ucap, 1),), SENTINEL, dtype=torch.int32, device="cuda") for _ in range(n)]
        self.dp = (C.c_void_p * max(n, 1))(*[t.data_ptr() for t in self.bufs])
        self.up = (C.c_void_p * max(n, 1))(*[t.data_ptr() for t in self.ubufs])
        torch.cuda.synchronize()

    def run(self, lens="opencv_fisheye", digital=None, **kw):
        a = dict(frames=self.frames.ctypes.data, ts=self.ts.ctypes.data, n=self.n, nw=self.nw.ctypes.data, nh=self.nh.ctypes.data,
                 dp=self.dp, up=self.up, dcap=self.dcap, ucap=self.ucap)
        a.update(kw)
        return self.dg._lib.gf_cuda_generate_stmaps_dev(self.dg._h, C.byref(self.dg.cp.c), abi.LENS[lens], abi.LENS[digital] if digital else 0, 1,
                                                        a["frames"], a["ts"], a["n"], a["nw"], a["nh"], a["dp"], a["up"], a["dcap"], a["ucap"], None)

    def untouched(self):
        import torch
        torch.cuda.synchronize()
        return all(bool((t == SENTINEL).all()) for t in self.bufs + self.ubufs)


@pytest.mark.gpu
def test_rejected_before_anything_is_enqueued():
    """n == 0, null arrays, capacities one float short, an unsupported lens pair and out-of-range sizes: the call returns the error and
    no buffer is written.  The faulty entry is the last one, so a call that validated frame by frame would have written the first."""
    sw, sh = STMAP_SIZE
    dg = g.DeviceGyro(make_cp(w=sw, h=sh))
    try:
        job = Job(dg)
        assert job.run(n=0) == GF_OK and job.run(n=0, frames=None, ts=None, nw=None, nh=None, dp=None, up=None) == GF_OK
        for field in ("frames", "ts", "nw", "nh", "dp", "up"):
            assert job.run(**{field: None}) == GF_ERR_BAD_PARAMS, field
        job.dp[job.n - 1] = None
        assert job.run() == GF_ERR_BAD_PARAMS
        job.dp[job.n - 1] = job.bufs[-1].data_ptr()
        assert job.run(dcap=job.dcap - 1) == GF_ERR_BUFFER_TOO_SMALL
        assert job.untouched()
        big = Job(dg, new_w=[sw, sw, sw + 9], new_h=[sh, sh, sh + 5])
        assert big.run(ucap=big.ucap - 1) == GF_ERR_BUFFER_TOO_SMALL
        assert big.run(lens="poly3", digital="gopro_superview") == GF_ERR_UNSUPPORTED_COMBO
        assert big.run(lens="gopro", digital="digital_stretch") == GF_ERR_UNSUPPORTED_COMBO        # the point path has it, the warp not
        assert big.untouched()
        for nw, nh, rc in ((3, sh, GF_ERR_SIZE_MISMATCH), (sw, 3, GF_ERR_SIZE_MISMATCH), (32769, 4, GF_ERR_SIZE_MISMATCH),
                           (4, 32769, GF_ERR_SIZE_MISMATCH), (16385, 4, GF_ERR_BAD_PARAMS)):
            bad = Job(dg, new_w=[sw, sw, nw], new_h=[sh, sh, nh])
            assert bad.run() == rc, (nw, nh)
            assert bad.untouched(), (nw, nh)
        assert job.run() == GF_OK and not job.untouched()            # the same arguments, corrected, do render
    finally:
        dg.close()


@pytest.mark.gpu
def test_sizes_errors_name_the_frame():
    """gf_cuda_stmap_sizes: n == 0 writes nothing; null arrays and unsupported pairs are refused; a frame whose undistorted size is out of
    range (its principal point far off the frame) fails the call with GF_ERR_SIZE_MISMATCH naming it, every size still written."""
    sw, sh = STMAP_SIZE
    lens_frames = [_scaled(LENS_A, sw, sh)] * 5
    # frame 3: an identity lens whose principal point is 1e5 px to the right moves every edge point ~1e5 px to the left
    far = dict(lens_frames[3], distortion_coeffs=[0.0] * 12); k = list(far["camera_matrix"]); k[2] = 1.0e5; far["camera_matrix"] = k
    lens_frames[3] = far
    dg = g.DeviceGyro(make_cp(w=sw, h=sh, lens_per_frame=lens_frames))
    lib = dg._lib
    try:
        nw = np.full(5, -7, np.int32); nh = np.full(5, -7, np.int32)
        fr = np.arange(5, dtype=np.uintp); ts = np.asarray(CLIP_TS)
        assert lib.gf_cuda_stmap_sizes(dg._h, C.byref(dg.cp.c), 1, 0, 1, fr.ctypes.data, ts.ctypes.data, 0, nw.ctypes.data, nh.ctypes.data, None) == GF_OK
        assert (nw == -7).all() and (nh == -7).all()
        for args in ((None, ts.ctypes.data, nw.ctypes.data, nh.ctypes.data), (fr.ctypes.data, None, nw.ctypes.data, nh.ctypes.data),
                     (fr.ctypes.data, ts.ctypes.data, None, nh.ctypes.data), (fr.ctypes.data, ts.ctypes.data, nw.ctypes.data, None)):
            assert lib.gf_cuda_stmap_sizes(dg._h, C.byref(dg.cp.c), 1, 0, 1, args[0], args[1], 5, args[2], args[3], None) == GF_ERR_BAD_PARAMS
        assert clip_sizes(dg, "poly3", "gopro_superview", True)[0] == GF_ERR_UNSUPPORTED_COMBO
        rc, nw, nh = clip_sizes(dg, "opencv_fisheye", None, True)
        assert rc == GF_ERR_SIZE_MISMATCH
        assert "frame 3" in lib.gf_cuda_last_error(None).decode()
        want = single_sizes(dg, "opencv_fisheye", None, True)
        assert [(r == GF_OK) for r, _, _ in want] == [True, True, True, False, True]
        assert [(w, h) for _, w, h in want] == list(zip(nw.tolist(), nh.tolist()))
        with pytest.raises(g.GyroflowCoreError) as e:
            dg.generate_stmaps("opencv_fisheye", None, CLIP_TS, CLIP_FRAMES)
        assert e.value.code == GF_ERR_SIZE_MISMATCH
        rc, nw, nh = clip_sizes(dg, "opencv_fisheye", None, True, frames=[0, 1, 2, 4], ts=[CLIP_TS[i] for i in (0, 1, 2, 4)])
        assert rc == GF_OK and [(w, h) for _, w, h in want[:3] + want[4:]] == list(zip(nw.tolist(), nh.tolist()))
    finally:
        dg.close()
