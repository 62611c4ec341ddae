"""The bookkeeping around the packed fisheye kernel's filtered rolling-shutter pre-pass (FilterPrepass in filter_prepass.cu; warp_kernel_x2.cuh:
the deferral in warp_x2_body and the tail branch of warp_kernel_x2): the deferred-pair queue and its inline fallback when it is full, the
tail launch's grid-stride loop, the ping-pong counters across frames of every kind, the per-context radial-table cache, and the ordering of
calls on one context that name different streams.

The tail renders deferred pairs exactly, so a broken queue mostly shows up as a slower kernel, not as wrong bytes.  Every frame here is
compared with the oracle byte for byte, and every path a test claims to reach is proven reached with the counts of gf_cuda_filter_stats
(CudaWrapper.filter_stats) or, for the overflow, with a host lower bound on the number of deferred pairs that needs no hook at all."""
import ctypes as C
import time

import numpy as np
import pytest

import gyroflow_b200 as g
from tests import cases, oracle_lib

QUEUE_CAP = 1 << 20
K_SMALLEST_CAP = [-0.25 / 0.5 ** 2 * 0.999, 0.0, 0.0, 0.0] + [0.0] * 8      # one-term lens at the smallest cap the filter accepts (0.5 rad)
K_BAND = [-0.42, 0.0, 0.0, 0.0] + [0.0] * 8                                # cap inside a 4K frame: a band of corners defers
K_NO_FILTER = [40.0, 0.0, 0.0, 0.0] + [0.0] * 8                            # conditioning cap below 0.5 rad: no filter


def radial_cap(k):
    """The r^2 cap the filter runs with for fisheye coefficients k[0..3], rounded to a table row as the warp rounds it (0: no filter)."""
    rows = np.zeros((8192, 4), np.float32)
    cap = C.c_float()
    assert g.load_library().gf_filter_radial_table((C.c_float * 4)(*k[:4]), rows.ctypes.data_as(C.c_void_p), 8192, C.byref(cap)) == 8192
    return cap.value


def pairs(p):
    return p.output_width * ((p.output_height + 1) // 2)


def deferred_pixels(p, m, cap):
    """Per output pixel of a full frame (identity rect maps): True where the filtered pre-pass cannot certify the pixel's row.  The
    reference's unfused _x, _y, _w of the middle matrix row in f32 (as the kernel computes them, bit for bit), then a = r^2 in f64: the
    divisor outside the exact sequences' window [2^-56, 2^48), or a at or above the cap with a margin of 2^-10 for the kernel's f32
    evaluation of a, whose table row there is NaN."""
    f = np.float32
    rm = np.asarray(m[p.matrix_count // 2], np.float32)
    pxs = (np.arange(p.output_width, dtype=np.float32) + f(p.translation2d[0]))[None, :]
    py = (np.arange(p.output_height, dtype=np.float32) + f(p.translation2d[1]))[:, None]
    _x = (pxs * rm[0] + py * rm[1]) + rm[2]
    _y = (pxs * rm[3] + py * rm[4]) + rm[5]
    _w = (pxs * rm[6] + py * rm[7]) + rm[8]
    w_ok = (_w >= f(2.0 ** -56)) & (_w < f(2.0 ** 48))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        w64 = _w.astype(np.float64)
        a = (_x / w64) ** 2 + (_y / w64) ** 2
    return ~w_ok | (a >= cap * (1.0 + 2.0 ** -10))


def deferral_lower_bound(p, m, cap):
    """Pixel pairs (x, y0), y0 even, that the main launch certainly defers: either pixel of the pair deferred (deferred_pixels)."""
    d = deferred_pixels(p, m, cap)
    if d.shape[0] % 2:
        d = np.vstack([d, np.zeros((1, d.shape[1]), bool)])
    return int((d[0::2] | d[1::2]).sum())


def test_lower_bound_against_a_direct_count():
    """The vectorised bound on a small frame against the same rule evaluated pixel by pixel with scalar f32 products and Python floats,
    on a frame where both clauses (divisor window, cap) decide some pixels."""
    p, src, m, mesh, dst0, pix, lens, digital = cases.build(dict(w=96, h=54, params=dict(k=K_BAND, translation2d=[3.5, -2.25]), fov=1.3))
    m = m.copy()
    m[p.matrix_count // 2, 6:9] = [np.float32(1e-3), np.float32(-2e-3), np.float32(0.04)]     # _w crosses zero inside the frame
    cap = radial_cap(list(p.k))
    assert cap > 0.0
    f = np.float32
    r = [f(v) for v in m[p.matrix_count // 2, :9]]
    want, n_w, n_a = 0, 0, 0
    for y0 in range(0, p.output_height, 2):
        for x in range(p.output_width):
            hit = False
            for y in (y0, y0 + 1):
                pxs, py = f(x) + f(p.translation2d[0]), f(y) + f(p.translation2d[1])
                _x, _y, _w = (pxs * r[0] + py * r[1]) + r[2], (pxs * r[3] + py * r[4]) + r[5], (pxs * r[6] + py * r[7]) + r[8]
                if not (2.0 ** -56 <= float(_w) < 2.0 ** 48):
                    hit = True; n_w += 1
                elif (float(_x) / float(_w)) ** 2 + (float(_y) / float(_w)) ** 2 >= cap * (1.0 + 2.0 ** -10):
                    hit = True; n_a += 1
            want += hit
    assert n_w > 0 and n_a > 0, (n_w, n_a)
    assert deferral_lower_bound(p, m, cap) == want
    assert 0 < want < pairs(p)


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------------


def _oracle(b):
    p, src, m, mesh, dst0, pix, lens, digital = b
    want = dst0.copy()
    assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
    return want


def _host_bufs(p, src, dst):
    return g.Buffers(g.BufferDescription((p.width, p.height, p.stride), src), g.BufferDescription((p.output_width, p.output_height, p.output_stride), dst))


def _dev_bufs(p, tsrc, tdst):
    return g.Buffers(g.BufferDescription((p.width, p.height, p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                     g.BufferDescription((p.output_width, p.output_height, p.output_stride), tdst.data_ptr(), length=tdst.numel()))


def _itm(b):
    return g.FrameTransform(matrices=b[2], kernel_params=b[0])


def _render(b, device, w=None):
    """One frame, HOST buffers or DEVICE buffers (host tables either way) on a fresh context (or `w`): (output, stats, launches)."""
    import torch
    p, src, m, mesh, dst0, pix, lens, digital = b
    if device:
        tsrc, tdst = torch.from_numpy(src).cuda(), torch.from_numpy(dst0.copy()).cuda()
        bufs = _dev_bufs(p, tsrc, tdst)
        torch.cuda.synchronize()
    else:
        got = dst0.copy()
        bufs = _host_bufs(p, src, got)
    own = w is None
    if own:
        w = g.CudaWrapper.new(p, pix, lens, digital, bufs)
    l0 = w.launch_count
    w.undistort_image(bufs, _itm(b))
    stats = w.filter_stats()                                    # waits for the context's streams
    launches = w.launch_count - l0
    if own:
        w.close()
    return (tdst.cpu().numpy() if device else got), stats, launches


def _render_planes(built, device):
    """Two planes of one geometry in one call (the fused coordinate pass); tables trusted either way: host tables are scanned on the
    host, device tables get a verdict word from gf_cuda_scan_tables_dev.  Returns ([outputs], stats, launches)."""
    import torch
    p0, _, m, _, _, pix, lens, digital = built[0]
    params = []
    for i, b in enumerate(built):
        p = b[0].copy(); p.plane_index = i; params.append(p)
    if device:
        keep = [(torch.from_numpy(b[1]).cuda(), torch.from_numpy(b[4].copy()).cuda()) for b in built]
        bufs = [_dev_bufs(params[i], s, d) for i, (s, d) in enumerate(keep)]
        tm = torch.from_numpy(m).cuda()
        flags = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        g.scan_tables_dev(tm.data_ptr(), m.shape[0], flags.data_ptr(), stream=torch.cuda.current_stream().cuda_stream or 1)
        torch.cuda.synchronize()
        assert int(flags.item()) == 0
    else:
        gots = [b[4].copy() for b in built]
        bufs = [_host_bufs(params[i], b[1], gots[i]) for i, b in enumerate(built)]
    w = g.CudaWrapper.new(params[0], pix, lens, digital, bufs[0])
    if device:
        w.undistort_planes_dev(bufs, params, tm.data_ptr(), m.shape[0], table_flags_dev=flags.data_ptr())
    else:
        w.undistort_planes(bufs, params, _itm(built[0]))
    stats = w.filter_stats()
    launches = w.launch_count
    w.close()
    return ([d.cpu().numpy() for _, d in keep] if device else gots), stats, launches


def _assert_same(want, got, what):
    n = int((want != got).sum())
    assert n == 0, "%s: %d mismatching bytes" % (what, n)


# (case, launches per frame: main + tail, plus the sampling pass of the two-pass path)
OVERFLOW = {
    "RGBA8": (dict(w=3840, h=2160, params=dict(k=K_SMALLEST_CAP)), 2),
    "Luma16": (dict(w=3840, h=2160, pix="Luma16", params=dict(k=K_SMALLEST_CAP), ts=2100.0), 2),
    "RGBAf": (dict(w=3840, h=2160, pix="RGBAf", params=dict(k=K_SMALLEST_CAP), ts=2900.0), 2),
    "bicubic": (dict(w=3840, h=2160, interp="Bicubic", params=dict(k=K_SMALLEST_CAP), ts=1500.0), 3),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(OVERFLOW) + ["planes"])
def test_overflow_falls_back_inline(name):
    """A frame that defers more pairs than the queue holds: the host bound alone proves the overflow, the hook's raw count agrees, and the
    pairs past the capacity are rendered inline by the main launch.  RGBA8 takes the hot interior block, Luma16 / RGBAf shade_lean,
    bicubic and the fused two-plane frame write coordinates (KV_PACKED_COORDS) for the sampling pass.  HOST and DEVICE buffers."""
    if name == "planes":
        case, n_launch = dict(w=3840, h=2160, pix="Luma8", params=dict(k=K_SMALLEST_CAP), ts=700.0), 4     # main + tail + two samplings
        built = [cases.build(dict(case, frame=i)) for i in range(2)]
        p, m = built[0][0], built[0][2]
        wants = []
        for i, b in enumerate(built):
            q = b[0].copy(); q.plane_index = i
            wants.append(_oracle((q,) + tuple(b[1:])))
    else:
        case, n_launch = OVERFLOW[name]
        b = cases.build(case)
        p, m = b[0], b[2]
        wants = [_oracle(b)]
    bound = deferral_lower_bound(p, m, radial_cap(list(p.k)))
    assert bound > QUEUE_CAP, bound                          # overflow proven without the hook
    for device in (False, True):
        if name == "planes":
            gots, s, launches = _render_planes(built, device)
        else:
            got, s, launches = _render(b, device)
            gots = [got]
        for i, (want, got) in enumerate(zip(wants, gots)):
            _assert_same(want, got, "%s device=%s plane %d" % (name, device, i))
        assert s["frames"] == 1 and s["cap"] == QUEUE_CAP, s
        assert bound <= s["count"] <= pairs(p), (bound, s)
        assert launches == n_launch, launches


@pytest.mark.gpu
def test_grid_stride_tail():
    """A frame that defers more pairs than the tail launch has threads (and fewer than the queue holds): the tail's grid-stride loop
    takes a second step, and every deferred pair is rendered."""
    b = cases.build(dict(w=3840, h=2160, params=dict(k=K_BAND), ts=1800.0))
    bound = deferral_lower_bound(b[0], b[2], radial_cap(list(b[0].k)))
    want = _oracle(b)
    for device in (False, True):
        got, s, launches = _render(b, device)
        _assert_same(want, got, "device=%s" % device)
        assert launches == 2 and s["frames"] == 1
        assert s["tail_threads"] < s["count"] < s["cap"], s
        assert s["count"] >= bound > 0, (bound, s)


@pytest.mark.gpu
def test_deferral_rate_and_guarded_path():
    """An ordinary 4K RGBA8 frame defers a small share of its pairs (a table of NaN, a counter that is never re-armed or a certificate
    that never passes would defer them all); the same frame from a DEVICE table without a verdict word runs the guarded path, which
    defers nothing but still launches main + tail."""
    import torch
    b = cases.build(dict(w=3840, h=2160, ts=2500.0))
    p, src, m, mesh, dst0, pix, lens, digital = b
    want = _oracle(b)
    got, s, launches = _render(b, False)
    _assert_same(want, got, "host")
    assert launches == 2 and s["frames"] == 1
    assert 0.001 < s["count"] / pairs(p) < 0.05, s["count"] / pairs(p)
    assert s["radial_builds"] == 1 and s["radial_hits"] == 0
    tsrc, tdst, tm = torch.from_numpy(src).cuda(), torch.from_numpy(dst0.copy()).cuda(), torch.from_numpy(m).cuda()
    bufs = _dev_bufs(p, tsrc, tdst)
    w = g.CudaWrapper.new(p, pix, lens, digital, bufs)
    torch.cuda.synchronize()
    w.undistort_image_dev(bufs, p, tm.data_ptr(), m.shape[0])
    s = w.filter_stats()
    assert w.launch_count == 2 and s["frames"] == 1 and s["count"] == 0, s
    _assert_same(want, tdst.cpu().numpy(), "guarded")
    w.close()


@pytest.mark.gpu
def test_counter_sequence_across_frame_kinds():
    """One context, one stream, no host sync: filtered frames mixed with an overflow frame, a frame without rolling shutter, a guarded
    frame (device table without a verdict: main + tail, nothing deferred) and a lens that runs without the filter.  Every frame equals the
    oracle, and in a second pass with a sync after each frame every filtered frame's count equals its count on a fresh context: the tail
    of each filtered frame re-arms the counter the next filtered frame uses, whatever ran in between."""
    import torch
    kinds = [("F", dict(ts=400.0)), ("O", dict(params=dict(k=K_SMALLEST_CAP), ts=900.0)), ("F", dict(ts=1300.0)), ("R", dict(rs=False, ts=1700.0)),
             ("F", dict(ts=2100.0)), ("G", dict(ts=2500.0)), ("F", dict(ts=2900.0)), ("N", dict(params=dict(k=K_NO_FILTER), ts=3300.0)), ("F", dict(ts=3600.0))]
    built = [cases.build(dict(w=3840, h=2160, **kw)) for _, kw in kinds]
    wants = [_oracle(b) for b in built]
    p, src, _, _, dst0, pix, lens, digital = built[0]
    tsrc = torch.from_numpy(src).cuda()
    outs = [torch.from_numpy(dst0.copy()).cuda() for _ in built]
    tms = [torch.from_numpy(b[2]).cuda() for b in built]
    w = g.CudaWrapper.new(p, pix, lens, digital, _dev_bufs(p, tsrc, outs[0]))
    torch.cuda.synchronize()

    def run(i):
        b = built[i]
        bufs = _dev_bufs(b[0], tsrc, outs[i])
        if kinds[i][0] == "G":
            w.undistort_image_dev(bufs, b[0], tms[i].data_ptr(), b[2].shape[0])
        else:
            w.undistort_image(bufs, _itm(b))

    for i in range(len(built)):
        run(i)
    w.synchronize()
    for i, want in enumerate(wants):
        _assert_same(want, outs[i].cpu().numpy(), "first pass, frame %d (%s)" % (i, kinds[i][0]))
    fresh = {i: _render(b, True)[1]["count"] for i, b in enumerate(built) if kinds[i][0] in "FO"}
    assert w.filter_stats()["count"] == fresh[len(built) - 1]
    assert fresh[1] > QUEUE_CAP and all(0 < fresh[i] < QUEUE_CAP for i in fresh if i != 1), fresh
    before = w.filter_stats()
    for i, (kind, _) in enumerate(kinds):
        outs[i].fill_(0xA5)
        torch.cuda.synchronize()
        run(i)
        s = w.filter_stats()
        assert s["frames"] - before["frames"] == (1 if kind in "FOG" else 0), (i, kind, s)
        want_count = fresh[i] if kind in "FO" else (0 if kind == "G" else before["count"])
        assert s["count"] == want_count, (i, kind, s["count"], want_count)
        _assert_same(wants[i], outs[i].cpu().numpy(), "second pass, frame %d (%s)" % (i, kind))
        before = s
    w.close()


LENSES = [[0.05, -0.01, 0.002, 0.0], [-0.05, 0.01, 0.0, 0.0], [0.12, -0.03, 0.004, -0.0005], [-0.1, 0.0, 0.002, 0.0],
          [0.2, -0.05, 0.0, 0.0], [-0.15, 0.02, 0.0, 0.0], [0.08, 0.0, -0.004, 0.0], [-0.02, -0.02, 0.0, 0.001],
          [0.15, 0.0, 0.0, -0.002], [-0.2, 0.04, 0.0, 0.0]]


@pytest.mark.gpu
def test_radial_table_lru():
    """Lens sequence A B C D A E B on one context: A is served from the cache, E evicts B (the least recently used entry, since A was used
    again) and B is rebuilt: 6 tables built, 1 lookup served from the cache, every frame equal to the oracle."""
    seq = [0, 1, 2, 3, 0, 4, 1]
    built = [cases.build(dict(w=640, h=360, params=dict(k=LENSES[j] + [0.0] * 8), ts=300.0 + 250.0 * i)) for i, j in enumerate(seq)]
    p, src, m, mesh, dst0, pix, lens, digital = built[0]
    got = dst0.copy()
    w = g.CudaWrapper.new(p, pix, lens, digital, _host_bufs(p, src, got))
    for i, b in enumerate(built):
        got[:] = b[4]
        w.undistort_image(_host_bufs(b[0], b[1], got), _itm(b))
        _assert_same(_oracle(b), got, "frame %d" % i)
    s = w.filter_stats()
    assert s["frames"] == 7 and s["radial_builds"] == 6 and s["radial_hits"] == 1, s
    w.close()


@pytest.mark.gpu
def test_radial_table_eviction_behind_a_gate():
    """Six frames with six new lenses queued behind a ~50 ms gate on a context whose four entries hold other lenses: the fifth and sixth
    evict entries whose first reader has not even uploaded its table yet.  The rebuild must wait for that reader (the pinned host copy
    it uploads from is overwritten by the rebuild): every frame equals the oracle."""
    import torch
    wb = [cases.build(dict(w=1280, h=720, params=dict(k=LENSES[j] + [0.0] * 8), ts=200.0 + 100.0 * j)) for j in range(4)]
    gb = [cases.build(dict(w=1280, h=720, params=dict(k=LENSES[4 + j] + [0.0] * 8), ts=800.0 + 300.0 * j)) for j in range(6)]
    p, src, m, mesh, dst0, pix, lens, digital = wb[0]
    tsrc = torch.from_numpy(src).cuda()
    outs = [torch.from_numpy(dst0.copy()).cuda() for _ in wb + gb]
    tms = [torch.from_numpy(b[2]).cuda() for b in wb + gb]
    flags = torch.full((len(tms),), -1, dtype=torch.int32, device="cuda")
    cur = torch.cuda.current_stream().cuda_stream or 1
    for i, tm in enumerate(tms):
        g.scan_tables_dev(tm.data_ptr(), tm.shape[0], flags[i:].data_ptr(), stream=cur)
    w = g.CudaWrapper.new(p, pix, lens, digital, _dev_bufs(p, tsrc, outs[0]))
    torch.cuda.synchronize()
    assert (flags.cpu() == 0).all()
    side = torch.cuda.Stream()

    def run(i, b):
        w.undistort_image_dev(_dev_bufs(b[0], tsrc, outs[i]), b[0], tms[i].data_ptr(), b[2].shape[0], stream=side.cuda_stream,
                              table_flags_dev=flags[i:].data_ptr())

    for i, b in enumerate(wb):                               # fill the four entries, allocate everything, then wait
        run(i, b)
    w.synchronize()
    gate_s = 0.05
    with torch.cuda.stream(side):
        torch.cuda._sleep(int(gate_s * 2.0e9))              # >= 50 ms at any SM clock up to 2 GHz
    t0 = time.perf_counter()
    for j, b in enumerate(gb):
        if j == 4:
            t_evict = time.perf_counter() - t0
        run(4 + j, b)
    w.synchronize()
    assert t_evict < 0.6 * gate_s, t_evict                  # the gate was still closed when the first eviction of a queued entry came
    for i, b in enumerate(wb + gb):
        _assert_same(_oracle(b), outs[i].cpu().numpy(), "frame %d" % i)
    s = w.filter_stats()
    assert s["frames"] == 10 and s["radial_builds"] == 10 and s["radial_hits"] == 0, s
    w.close()


# frames of the two-stream test: lens per frame, so that consecutive frames (on different streams) share the lens or not
TWO_STREAM_LENSES = [0, 1, 1, 0, 0, 2, 2, 1]


def two_stream_frames():
    return [cases.build(dict(w=1920, h=1080, params=dict(k=LENSES[j] + [0.0] * 8), ts=300.0 + 410.0 * i)) for i, j in enumerate(TWO_STREAM_LENSES)]


def render_on_two_streams(built, gate_s=0.05):
    """Frames alternating between two streams on one context (DEVICE buffers, device tables with verdict words), both streams released
    together from one gate event so that consecutive frames' launches can overlap.  Returns (context, streams, outputs, keep-alive)."""
    import torch
    p, src, m, mesh, dst0, pix, lens, digital = built[0]
    tsrc = torch.from_numpy(src).cuda()
    outs = [torch.from_numpy(dst0.copy()).cuda() for _ in built]
    tms = [torch.from_numpy(b[2]).cuda() for b in built]
    flags = torch.full((len(built),), -1, dtype=torch.int32, device="cuda")
    cur = torch.cuda.current_stream().cuda_stream or 1
    for i, tm in enumerate(tms):
        g.scan_tables_dev(tm.data_ptr(), tm.shape[0], flags[i:].data_ptr(), stream=cur)
    w = g.CudaWrapper.new(p, pix, lens, digital, _dev_bufs(p, tsrc, outs[0]))
    torch.cuda.synchronize()
    assert (flags.cpu() == 0).all()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]

    def run(i):
        b = built[i]
        w.undistort_image_dev(_dev_bufs(b[0], tsrc, outs[i]), b[0], tms[i].data_ptr(), b[2].shape[0], stream=streams[i % 2].cuda_stream,
                              table_flags_dev=flags[i:].data_ptr())

    for j in sorted(set(TWO_STREAM_LENSES)):                # every lens's table and the queue allocated before the gate: nothing below
        run(TWO_STREAM_LENSES.index(j))                     # allocates (an allocation may wait for the device)
    w.synchronize()
    for o in outs:                                          # back to the sentinel: a pair the gated run misses must show
        o.fill_(0xA5)
    torch.cuda.synchronize()
    gate = torch.cuda.Stream()
    with torch.cuda.stream(gate):
        torch.cuda._sleep(int(gate_s * 2.0e9))
    ev = torch.cuda.Event()
    ev.record(gate)
    for s in streams:
        s.wait_event(ev)
    for i in range(len(built)):
        run(i)
    return w, streams, outs, run, (tsrc, tms, flags, gate)


@pytest.mark.gpu
def test_two_streams_one_context():
    """Calls on one context that name different streams are ordered after one another: frames alternating between two streams, released
    together, all equal the oracle (the deferred-pair queue, its counters and the staging are shared by the context's calls);
    synchronize() covers both streams; each frame's deferral count, re-rendered with a sync after it, equals its count on a fresh context.
    Without the ordering, consecutive frames' main launches append to the shared queue at once and the tail of one re-arms the counter
    the other is appending to: 442,631 of the frames' bytes kept the sentinel on an H100."""
    import torch
    built = two_stream_frames()
    wants = [_oracle(b) for b in built]
    w, streams, outs, run, keep = render_on_two_streams(built)
    w.synchronize()
    assert all(s.query() for s in streams)                  # the last call's stream is ordered after every earlier call
    last = w.filter_stats()["count"]
    bad = [(i, int((want != outs[i].cpu().numpy()).sum())) for i, want in enumerate(wants)]
    assert all(n == 0 for _, n in bad), bad
    fresh = [_render(b, True)[1]["count"] for b in built]
    assert last == fresh[-1], (last, fresh)
    for i in range(len(built)):
        outs[i].fill_(0xA5)
        torch.cuda.synchronize()
        run(i)
        assert w.filter_stats()["count"] == fresh[i], (i, fresh)
        _assert_same(wants[i], outs[i].cpu().numpy(), "second pass, frame %d" % i)
    w.close()
