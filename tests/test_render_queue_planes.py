"""Multi-plane decoder frames through the render queue (gf_cuda_queue_create_planes / gf_cuda_queue_submit_planes): one producer launch
per frame, every plane warped from that one table, one checksum launch over all planes.

The per-plane yardstick is the reference's render loop (rendering/mod.rs:483-548) spelled out with the existing single-plane calls:
the frame's table (the device producer's, read back — the one the queue warps with; tests/test_render_queue.py pins it to the host
producer), gf_get_frame_transform_at with each plane's buffers, pixel_value_limit / max_pixel_value / plane_index / FILL_WITH_BACKGROUND
as the render loop sets them, then gf_cuda_undistort_image and the CPU oracle on that plane.  Launch counts are derived from the same
plane groups rendered through gf_cuda_undistort_planes_dev_flagged on one context."""
import ctypes as C
import os
import socket

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi, render_queue
from gyroflow_b200 import synth
from gyroflow_b200.render_queue import checksum_host, checksum_planes_host, layout
from tests import cases, oracle_lib

FPS = 60.0
LAYOUTS = ["nv12", "nv21", "p010", "yuv420p", "yuv422p16", "yuv444p10", "yuva444p12", "gbrapf32", "gbrpf32"]


def _bpp(pix):
    _, count, sdt = abi.PIXEL_TYPES[pix]
    return count * np.dtype(sdt).itemsize


# ---------------------------------------------------------------------------------------------------------------- CPU-only
def test_queue_plane_struct_matches_the_library():
    lib = abi.load_library()
    assert C.sizeof(abi.QueuePlane) == 32 and C.sizeof(abi.ChecksumPlane) == 32
    assert [getattr(abi.QueuePlane, f).offset for f in ("pixel_type", "w_div", "h_div", "max_value", "background")] == [0, 4, 8, 12, 16]
    assert [getattr(abi.ChecksumPlane, f).offset for f in ("ptr", "row_bytes", "stride", "rows")] == [0, 8, 16, 24]
    assert lib.gf_abi_struct_size(11) == C.sizeof(abi.QueuePlane)
    assert lib.gf_abi_struct_size(12) == C.sizeof(abi.ChecksumPlane)


# format -> [(pixel type, w_div, h_div, max value, components)], as create_planes_proc! lists them (rendering/mod.rs:563-651)
TABLE = {
    "nv12": [("Luma8", 1, 1, 255.0, (0,)), ("UV8", 2, 2, 255.0, (1, 2))],
    "nv21": [("Luma8", 1, 1, 255.0, (0,)), ("UV8", 2, 2, 255.0, (2, 1))],
    "yuv420p": [("Luma8", 1, 1, 255.0, (0,)), ("Luma8", 2, 2, 255.0, (1,)), ("Luma8", 2, 2, 255.0, (2,))],
    "yuvj420p": [("Luma8", 1, 1, 255.0, (0,)), ("Luma8", 2, 2, 255.0, (1,)), ("Luma8", 2, 2, 255.0, (2,))],
    "gbrapf32": [("R32f", 1, 1, 255.0, (2,)), ("R32f", 1, 1, 255.0, (0,)), ("R32f", 1, 1, 255.0, (1,)), ("R32f", 1, 1, 255.0, (3,))],
    "gbrpf32": [("R32f", 1, 1, 255.0, (2,)), ("R32f", 1, 1, 255.0, (0,)), ("R32f", 1, 1, 255.0, (1,))],
}
for _s, _d in (("0", (2, 2)), ("2", (2, 1)), ("4", (1, 1))):
    for _b in ("10", "16"):
        TABLE["p%s%s" % (_s, _b)] = [("Luma16", 1, 1, 65535.0, (0,)), ("UV16", _d[0], _d[1], 65535.0, (1, 2))]
for _s, _d in (("20", (2, 2)), ("22", (2, 1)), ("44", (1, 1))):
    for _b, _m in (("10", 1023.0), ("12", 4095.0), ("14", 16383.0), ("16", 65535.0)):
        TABLE["yuv4%sp%s" % (_s, _b)] = [("Luma16", 1, 1, _m, (0,))] + [("Luma16", _d[0], _d[1], _m, (c,)) for c in (1, 2)]
for _b, _m in (("10", 1023.0), ("12", 4095.0), ("16", 65535.0)):
    TABLE["yuva444p%s" % _b] = [("Luma16", 1, 1, _m, (c,)) for c in range(4)]


def test_decoder_format_table():
    assert set(render_queue.DECODER_FORMATS) == set(TABLE)
    for fmt, want in TABLE.items():
        got = layout(fmt, 1921, 1081)
        assert [(p.pixel_type, p.w_div, p.h_div, p.max_value, p.components) for p, _ in got] == want, fmt
        for (p, (w, h)), (_, wd, hd, _, _) in zip(got, want):
            assert (w, h) == (-(-1921 // wd), -(-1081 // hd)), fmt         # ffmpeg's chroma size: AV_CEIL_RSHIFT
    assert [s for _, s in layout("P010LE", 7, 5)] == [(7, 5), (4, 3)]
    c = layout("nv12", 8, 8)[1][0].to_c((0.5, 0.25, 0.0, 1.0))
    assert (c.pixel_type, c.w_div, c.h_div, c.max_value, list(c.background)) == (abi.PIXEL_TYPES["UV8"][0], 2, 2, 255.0, [0.5, 0.25, 0.0, 1.0])
    with pytest.raises(KeyError):
        layout("bgr0", 8, 8)


def _direct_checksum(data: bytes) -> int:
    """sum(word[i] * (2 i + 1)) mod 2^64 byte by byte: byte g adds b * 256^(g % 4) * (2 (g // 4) + 1); a last partial word is left out."""
    s = 0
    for gi in range(len(data) // 4 * 4):
        s += data[gi] * (256 ** (gi % 4)) * (2 * (gi // 4) + 1)
    return s % (1 << 64)


def test_multi_plane_checksum_host_restatement():
    rng = np.random.default_rng(5)
    bufs = [rng.integers(0, 256, n, dtype=np.uint8) for n in (1000, 777, 64, 333)]
    # odd strides, row lengths that are no multiple of 4, a descriptor with padding skipped and one with zero rows
    descs = [(bufs[0], 13, 17, 41), (bufs[1], 7, 7, 100), (bufs[2], 0, 8, 5), (bufs[3], 30, 33, 10)]
    cat = b"".join(bytes(render_queue.plane_rows(b, rb, st, r)) for b, rb, st, r in descs)
    assert len(cat) == 13 * 41 + 7 * 100 + 30 * 10
    assert checksum_planes_host(descs) == _direct_checksum(cat)
    # one descriptor of whole rows is the one-plane checksum of the buffer
    buf = rng.integers(0, 256, 37 * 11, dtype=np.uint8)
    assert checksum_planes_host([(buf, 37, 37, 11)]) == checksum_host(buf) == _direct_checksum(bytes(buf))
    # the words run across descriptors: splitting one buffer into two descriptors changes nothing
    assert checksum_planes_host([(buf, 37, 37, 5), (buf[5 * 37:], 37, 37, 6)]) == checksum_host(buf)


def _cfg(p, lens="opencv_fisheye", digital=None, depth=2, checksum=True):
    cfg = abi.QueueConfig()
    cfg.device, cfg.distortion_model, cfg.digital_lens = 0, abi.LENS[lens], abi.LENS[digital] if digital else 0
    cfg.depth, cfg.pin_numa, cfg.checksum = depth, 0, int(checksum)
    cfg.stab = g.stab_config(p, "Luma8", digital_lens=digital)
    return cfg


def _protos(fmt, w, h, kind="host"):
    ins, outs, keep = [], [], []
    for pl, (pw, ph) in layout(fmt, w, h):
        st = pw * _bpp(pl.pixel_type)
        for lst in (ins, outs):
            a = np.zeros(st * ph, np.uint8); keep.append(a)
            d = g.BufferDescription((pw, ph, st), a) if kind == "host" else g.BufferDescription((pw, ph, st), 0x10000, length=st * ph)
            lst.append(d.to_c())
    return ins, outs, keep


def _create(cfg, cp, planes, ins, outs):
    lib = abi.load_library()
    n = len(planes)
    h = C.c_void_p()
    rc = lib.gf_cuda_queue_create_planes(C.byref(h), C.byref(cfg), C.byref(cp.c), n, (abi.QueuePlane * max(n, 1))(*planes),
                                         (abi.BufferDesc * max(n, 1))(*ins), (abi.BufferDesc * max(n, 1))(*outs))
    return rc, h, (lib.gf_cuda_last_error(None) or b"").decode()


def test_create_planes_validation_fails_before_any_cuda_call():
    """Every rejected layout fails with GF_ERR_BAD_PARAMS and names the plane — before the device is touched, so also without one."""
    w, h = 64, 48
    p = synth.base_kernel_params(w, h, pixel_type="Luma8")
    org, sm = cases.gyro()
    cp = g.ComputeParams(p, org, sm)
    nv12 = [pl.to_c() for pl, _ in layout("nv12", w, h)]
    ins, outs, keep = _protos("nv12", w, h)

    rc, q, msg = _create(_cfg(p), cp, [], [], [])
    assert rc == -1 and not q.value and "n_planes" in msg
    five = [nv12[0]] * 5
    rc, _, msg = _create(_cfg(p), cp, five, [ins[0]] * 5, [outs[0]] * 5)
    assert rc == -1 and "n_planes" in msg

    bad = [abi.QueuePlane.from_buffer_copy(x) for x in nv12]; bad[1].h_div = 3
    rc, _, msg = _create(_cfg(p), cp, bad, ins, outs)
    assert rc == -1 and msg.startswith("plane 1:") and "w_div" in msg

    narrow = [abi.BufferDesc.from_buffer_copy(x) for x in ins]; narrow[1].width = w // 2 - 1   # UV8 must be ceil(W / 2) wide
    rc, _, msg = _create(_cfg(p), cp, nv12, narrow, outs)
    assert rc == -1 and msg.startswith("plane 1:") and "UV" in msg
    narrow_out = [abi.BufferDesc.from_buffer_copy(x) for x in outs]; narrow_out[1].width = w // 2 + 1
    rc, _, msg = _create(_cfg(p), cp, nv12, ins, narrow_out)
    assert rc == -1 and msg.startswith("plane 1:")

    dins, douts, _ = _protos("nv12", w, h, kind="device")
    rc, _, msg = _create(_cfg(p), cp, nv12, [ins[0], dins[1]], [outs[0], douts[1]])     # HOST luma, DEVICE chroma
    assert rc == -1 and msg.startswith("plane 1:") and "HOST" in msg
    rc, _, msg = _create(_cfg(p), cp, nv12, ins, [outs[0], douts[1]])
    assert rc == -1 and msg.startswith("plane 1:")

    short = [abi.BufferDesc.from_buffer_copy(x) for x in outs]; short[0].len -= 1      # output must hold height full rows
    rc, _, msg = _create(_cfg(p), cp, nv12, ins, short)
    assert rc == -1 and msg.startswith("plane 0:")

    # no kernel for this lens as the main model (gf_combo_supported says so on the host)
    assert abi.load_library().gf_combo_supported(abi.PIXEL_TYPES["Luma8"][0], abi.LENS["gopro_superview"], 0, 2) == 0
    rc, _, msg = _create(_cfg(p, lens="gopro_superview"), cp, nv12, ins, outs)
    assert rc == -1 and msg.startswith("plane 0:")
    unknown = [abi.QueuePlane.from_buffer_copy(x) for x in nv12]; unknown[1].pixel_type = 99
    rc, _, msg = _create(_cfg(p), cp, unknown, ins, outs)
    assert rc == -1 and msg.startswith("plane 1:")
    del keep


def test_submit_planes_null_queue():
    lib = abi.load_library()
    d = (abi.BufferDesc * 1)()
    assert lib.gf_cuda_queue_submit_planes(None, 0, 0.0, 1, d, d, None, 0, 0) == -1


# ---------------------------------------------------------------------------------------------------------------- GPU
class _Job:
    """A small decoder job of format `fmt`: frame size W x H, per-plane sources and buffers, the queue and the yardsticks."""

    def __init__(self, fmt, w=318, h=182, lens="opencv_fisheye", digital=None, interpolation="Bilinear", bg_mode=0, n=4, kind="device",
                 cpkw=None):
        import torch
        self.fmt, self.w, self.h, self.lens, self.digital, self.n, self.kind = fmt, w, h, lens, digital, n, kind
        self.planes = layout(fmt, w, h)
        self.p = synth.base_kernel_params(w, h, pixel_type=self.planes[0][0].pixel_type, lens=lens, digital_lens=digital, interpolation=interpolation)
        self.p.background_mode = bg_mode
        org, sm = synth.synthetic_gyro(n / FPS + 2.0)
        self.cp = g.ComputeParams(self.p, org, sm, **(cpkw or {}))
        if bg_mode == 3:
            self.cp.c.background_margin, self.cp.c.background_margin_feather = 0.1, 0.05
        self.st = g.stab_config(self.p, self.planes[0][0].pixel_type, digital_lens=digital)
        self.bgs = [(0.1 + 0.2 * i, 0.7 - 0.1 * i, 0.3, 1.0) for i in range(len(self.planes))]
        self.specs = [pl.to_c(bg) for (pl, _), bg in zip(self.planes, self.bgs)]
        # odd strides on purpose: input rows padded by 8 bytes, output rows by 4 (an odd stride for the 8-bit chroma of odd widths)
        self.geo = [(pw, ph, pw * _bpp(pl.pixel_type) + 8, pw * _bpp(pl.pixel_type) + 4) for pl, (pw, ph) in self.planes]
        self.srcs = [[synth.synthetic_frame(pw, ph, pl.pixel_type, frame=f * 7 + i, stride=si)
                      for i, ((pl, _), (pw, ph, si, so)) in enumerate(zip(self.planes, self.geo))] for f in range(2)]
        if kind == "device":
            self.tsrc = [[torch.from_numpy(s).cuda() for s in fs] for fs in self.srcs]
            self.outs = [[torch.zeros(ph * so, dtype=torch.uint8, device="cuda") for (pw, ph, si, so) in self.geo] for _ in range(n)]
        else:
            self.tsrc = [[torch.from_numpy(s).pin_memory() for s in fs] for fs in self.srcs]
            self.outs = [[torch.zeros(ph * so, dtype=torch.uint8).pin_memory() for (pw, ph, si, so) in self.geo] for _ in range(n)]

    def _desc(self, t, size):
        return g.BufferDescription(size, t.numpy()) if self.kind == "host" else g.BufferDescription(size, t.data_ptr(), length=t.numel())

    def buffers(self, f):
        return [g.Buffers(self._desc(self.tsrc[f % 2][i], (pw, ph, si)), self._desc(self.outs[f][i], (pw, ph, so)))
                for i, (pw, ph, si, so) in enumerate(self.geo)]

    def ts(self, f):
        return 300.0 + f * (1000.0 / FPS)

    def queue(self, depth=3, checksum=True):
        b = self.buffers(0)
        return g.RenderQueue.for_planes(self.cp, self.st, self.lens, self.digital, self.specs, [x.input for x in b], [x.output for x in b],
                                        depth=depth, checksum=checksum)

    def plane_stab(self, i):
        s = abi.StabConfig.from_buffer_copy(self.st)
        s.pixel_type = abi.PIXEL_TYPES[self.planes[i][0].pixel_type][0]
        s.background[:] = list(self.bgs[i])
        return s

    def frame_params(self, dg, mats, f, fill, flags_dev=0):
        """The frame's table (device producer, read back) and every plane's KernelParams as the render loop completes them."""
        kp0, rows, _, mfov = dg.frame_transform(self.ts(f), mats.data_ptr(), mats.shape[0], frame=f, table_flags_dev=flags_dev, with_fov=True)
        table = mats.cpu().numpy()[:rows].copy()
        kps = []
        for i, (pl, _) in enumerate(self.planes):
            kp = kp0.copy()
            g.get_frame_transform_at(self.plane_stab(i), self.cp, self.buffers(f)[i], kp, frame=f, minimal_fov=mfov, timestamp_ms=self.ts(f))
            kp.pixel_value_limit = kp.max_pixel_value = pl.max_value
            kp.plane_index = i
            if fill:
                kp.flags |= abi.FLAG_FILL_WITH_BACKGROUND
            kps.append(kp)
        return table, rows, kps

    def groups(self):
        out = {}
        for i, (pl, _) in enumerate(self.planes):
            out.setdefault((pl.pixel_type, pl.w_div, pl.h_div), []).append(i)
        return list(out.values())


def _got(job, f, i):
    return job.outs[f][i].cpu().numpy() if job.kind == "device" else job.outs[f][i].numpy().copy()


def _check_job(job, fill=False, depth=3, launches=True):
    """Render job.n frames through the queue, then check every plane of every frame against the per-plane calls and the oracle, the
    frame checksum against the host restatement, and (DEVICE) the queue's launch count against the same groups on one context."""
    import torch
    q = job.queue(depth=depth)
    sums = q.render(range(job.n), job.ts, job.buffers, fill_with_background=fill)
    n_launch = q.launch_count
    q.close()
    assert list(sums) == list(range(job.n))
    dg = g.DeviceGyro(job.cp)
    rows_max = max(job.w, job.h)
    mats = torch.zeros((rows_max, 14), dtype=torch.float32, device="cuda")
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    wrappers, group_ctx, want_launches = {}, {}, 0
    for f in range(job.n):
        table, rows, kps = job.frame_params(dg, mats, f, fill, flags.data_ptr())
        descs = []
        for i, (pl, _) in enumerate(job.planes):
            pw, ph, si, so = job.geo[i]
            src = job.srcs[f % 2][i]
            want = np.zeros(ph * so, np.uint8)
            assert oracle_lib.undistort_image(src, want, kps[i], pl.pixel_type, job.lens, job.digital, table) == 0
            per_plane = np.zeros(ph * so, np.uint8)
            bh = g.Buffers(g.BufferDescription((pw, ph, si), src), g.BufferDescription((pw, ph, so), per_plane))
            if i not in wrappers:
                wrappers[i] = g.CudaWrapper.new(kps[i], pl.pixel_type, job.lens, job.digital, bh)
            wrappers[i].undistort_image(bh, g.FrameTransform(matrices=table, kernel_params=kps[i]))
            got = _got(job, f, i)
            assert np.array_equal(per_plane, want), (job.fmt, f, i, "per-plane call vs oracle")
            assert np.array_equal(got, want), (job.fmt, f, i, "queue vs oracle")
            descs.append((got, so, so, ph))
        assert sums[f] == checksum_planes_host(descs), (job.fmt, f)
        if launches and job.kind == "device":
            # the same plane groups through gf_cuda_undistort_planes_dev_flagged on one context, same table and verdict word
            for grp in job.groups():
                k = grp[0]
                bufs = [job.buffers(f)[i] for i in grp]
                if k not in group_ctx:
                    group_ctx[k] = g.CudaWrapper.new(kps[k], job.planes[k][0].pixel_type, job.lens, job.digital, bufs[0])
                scratch = [torch.zeros_like(job.outs[f][i]) for i in grp]
                sb = [g.Buffers(b.input, g.BufferDescription(b.output.size, t.data_ptr(), length=t.numel())) for b, t in zip(bufs, scratch)]
                l0 = group_ctx[k].launch_count
                group_ctx[k].undistort_planes_dev(sb, [kps[i] for i in grp], mats.data_ptr(), rows, table_flags_dev=flags.data_ptr())
                group_ctx[k].synchronize()
                want_launches += group_ctx[k].launch_count - l0
                for i, t in zip(grp, scratch):
                    assert np.array_equal(t.cpu().numpy(), _got(job, f, i)), (job.fmt, f, i, "planes call vs queue")
            want_launches += 2                       # one producer launch and one checksum launch per frame
    if launches and job.kind == "device":
        assert n_launch == want_launches, (job.fmt, n_launch, want_launches)
    for w in list(wrappers.values()) + list(group_ctx.values()):
        w.close()
    dg.close()
    return sums, n_launch


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["device", "host"])
@pytest.mark.parametrize("fmt", LAYOUTS)
def test_planes_queue_matches_per_plane_calls_and_oracle(fmt, kind):
    _check_job(_Job(fmt, kind=kind, n=4), depth=3)


@pytest.mark.gpu
@pytest.mark.parametrize("interp,fill,bg_mode", [
    ("Bilinear", True, 0),
    ("Lanczos4", False, 0),
    ("Lanczos4", True, 0),
    ("EWA: Robidoux", False, 0),
    ("Bilinear", False, 3),                   # margin + feather on the chroma planes too
])
def test_planes_queue_resamplers_and_background(interp, fill, bg_mode):
    _check_job(_Job("yuv420p", interpolation=interp, bg_mode=bg_mode, n=3), fill=fill, depth=2)


@pytest.mark.gpu
def test_planes_share_one_producer_and_one_coordinate_pass():
    """Structural facts behind the launch counts: a U+V (or GBRAPF32) group is one coordinate pass plus one sampling pass per plane, and a
    frame has one producer launch whatever its plane count."""
    import torch
    for fmt, grp_planes in (("yuv420p", [1, 2]), ("gbrapf32", [0, 1, 2, 3])):
        job = _Job(fmt, n=1)
        dg = g.DeviceGyro(job.cp)
        mats = torch.zeros((max(job.w, job.h), 14), dtype=torch.float32, device="cuda")
        flags = torch.zeros(1, dtype=torch.int32, device="cuda")
        table, rows, kps = job.frame_params(dg, mats, 0, False, flags.data_ptr())
        bufs = job.buffers(0)
        ctx = g.CudaWrapper.new(kps[grp_planes[0]], job.planes[grp_planes[0]][0].pixel_type, job.lens, None, bufs[grp_planes[0]])
        l0 = ctx.launch_count
        ctx.undistort_planes_dev([bufs[i] for i in grp_planes], [kps[i] for i in grp_planes], mats.data_ptr(), rows, table_flags_dev=flags.data_ptr())
        fused = ctx.launch_count - l0
        l0 = ctx.launch_count
        ctx.undistort_planes_dev([bufs[grp_planes[0]]], [kps[grp_planes[0]]], mats.data_ptr(), rows, table_flags_dev=flags.data_ptr())
        single = ctx.launch_count - l0                           # bilinear, one plane: the warp alone (main launch + filter tail, if any)
        ctx.synchronize(); ctx.close(); dg.close()
        # one coordinate pass (planned like the lone warp: main launch + filter tail, if any) + one sampling pass per plane
        assert fused == single + len(grp_planes), (fmt, fused, single)
        q = job.queue(depth=1)
        q.render([0], job.ts, job.buffers)
        per_frame = q.launch_count
        q.close()
        others = 0 if fmt == "gbrapf32" else single              # yuv420p: the luma plane's own warp, the same plan as a lone chroma plane
        assert per_frame == 1 + others + fused + 1, (fmt, per_frame)


@pytest.mark.gpu
def test_one_plane_layout_is_the_single_plane_queue():
    """A one-plane RGBA8 layout: the same bytes, launch count and checksums as a gf_cuda_queue_create queue on the same frames."""
    import torch
    w, h, n = 320, 180, 5
    p = synth.base_kernel_params(w, h, pixel_type="RGBA8")
    org, sm = cases.gyro()
    cp = g.ComputeParams(p, org, sm)
    st = g.stab_config(p, "RGBA8")
    src = torch.from_numpy(synth.synthetic_frame(w, h, "RGBA8", stride=p.stride)).cuda()
    outs = {k: [torch.zeros((h, p.output_stride), dtype=torch.uint8, device="cuda") for _ in range(n)] for k in ("one", "planes")}
    mk = lambda k, f: g.Buffers(g.BufferDescription((w, h, p.stride), src.data_ptr(), length=src.numel()),
                                g.BufferDescription((w, h, p.output_stride), outs[k][f].data_ptr(), length=outs[k][f].numel()))
    ts = lambda f: 400.0 + f * (1000.0 / FPS)
    q1 = g.RenderQueue(cp, st, "opencv_fisheye", None, mk("one", 0).input, mk("one", 0).output, depth=3, checksum=True)
    s1 = q1.render(range(n), ts, lambda f: mk("one", f)); l1 = q1.launch_count; q1.close()
    spec = render_queue.PlaneLayout("RGBA8", 1, 1, 255.0, ()).to_c()
    q2 = g.RenderQueue.for_planes(cp, st, "opencv_fisheye", None, [spec], [mk("planes", 0).input], [mk("planes", 0).output], depth=3, checksum=True)
    s2 = q2.render(range(n), ts, lambda f: [mk("planes", f)]); l2 = q2.launch_count; q2.close()
    assert s1 == s2 and l1 == l2
    for f in range(n):
        a, b = outs["one"][f].cpu().numpy(), outs["planes"][f].cpu().numpy()
        assert np.array_equal(a, b), f
        assert s1[f] == checksum_host(a)


@pytest.mark.gpu
def test_submit_planes_validation():
    job = _Job("nv12", n=2)
    q = job.queue(depth=2)
    b = job.buffers(0)
    lib = q._lib
    def submit(bufs, n=None):
        n = len(bufs) if n is None else n
        ins = (abi.BufferDesc * len(bufs))(*[x.input.to_c() for x in bufs])
        outs = (abi.BufferDesc * len(bufs))(*[x.output.to_c() for x in bufs])
        rc = lib.gf_cuda_queue_submit_planes(q._h, 0, 300.0, n, ins, outs, None, 0, 0)
        return rc, (lib.gf_cuda_queue_last_error(q._h) or b"").decode()
    rc, msg = submit(b[:1])
    assert rc == -1 and "n_planes" in msg
    wrong = [b[0], g.Buffers(b[1].input, g.BufferDescription((b[1].output.size[0], b[1].output.size[1], b[1].output.size[2] + 4),
                                                             b[1].output.data, length=b[1].output.length))]
    rc, msg = submit(wrong)
    assert rc == -1 and msg.startswith("plane 1:")
    host = np.zeros(b[1].input.length, np.uint8)
    mixed = [b[0], g.Buffers(g.BufferDescription(b[1].input.size, host), b[1].output)]
    rc, msg = submit(mixed)
    assert rc == -1 and msg.startswith("plane 1:") and "HOST" in msg
    rc = lib.gf_cuda_queue_submit(q._h, 0, 300.0, C.byref(b[0].input.to_c()), C.byref(b[0].output.to_c()), None, 0)
    assert rc == -1                                            # a planes queue takes the planes submit
    assert q.launch_count == 0                                 # nothing was enqueued
    q.render([0, 1], job.ts, job.buffers)                      # and the queue still works
    q.close()


@pytest.mark.gpu
def test_checksum_kernel_odd_strides_and_rows():
    """gf_cuda_checksum_planes_dev (one launch) against the host restatement: unaligned pointers, odd strides, odd row lengths."""
    import torch
    lib = abi.load_library()
    rng = np.random.default_rng(11)
    host = [rng.integers(0, 256, n, dtype=np.uint8) for n in (5003, 4096, 999, 12345)]
    dev = [torch.from_numpy(a).cuda() for a in host]
    out = torch.zeros(1, dtype=torch.int64, device="cuda")
    cases_ = [
        [(0, 1, 13, 17, 41), (1, 0, 7, 7, 100), (2, 3, 30, 33, 10), (3, 2, 101, 103, 90)],
        [(1, 0, 4096, 4096, 1)],
        [(0, 1, 5001, 5001, 1), (3, 5, 3, 4, 1000)],
        [(2, 0, 0, 8, 9), (1, 0, 2, 2, 1)],                    # 2 bytes in all: no whole word, checksum 0
    ]
    for descs in cases_:
        arr = (abi.ChecksumPlane * len(descs))()
        for k, (b, off, rb, st, r) in enumerate(descs):
            arr[k].ptr, arr[k].row_bytes, arr[k].stride, arr[k].rows = dev[b].data_ptr() + off, rb, st, r
        assert lib.gf_cuda_checksum_planes_dev(arr, len(descs), out.data_ptr(), None) == 0
        torch.cuda.synchronize()
        want = checksum_planes_host([(host[b][off:], rb, st, r) for b, off, rb, st, r in descs])
        assert (int(out.item()) & ((1 << 64) - 1)) == want, descs
    # one whole-row descriptor equals gf_cuda_checksum_dev of the same bytes
    one = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.gf_cuda_checksum_dev(dev[1].data_ptr(), 4096, one.data_ptr(), None) == 0
    arr = (abi.ChecksumPlane * 1)(); arr[0].ptr, arr[0].row_bytes, arr[0].stride, arr[0].rows = dev[1].data_ptr(), 64, 64, 64
    assert lib.gf_cuda_checksum_planes_dev(arr, 1, out.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert int(out.item()) == int(one.item())
    assert lib.gf_cuda_checksum_planes_dev(arr, 5, out.data_ptr(), None) == -1


@pytest.mark.gpu
def test_cfg3_8k_yuv422p16_through_the_queue():
    """BASELINE cfg 3 at full size: an 8K YUV422P16 frame, opencv_fisheye + gopro_superview, rolling shutter on, through the queue; every
    plane's checksum against the oracle's render of that plane, and the frame checksum against the planes together."""
    import torch
    w, h = 7680, 4320
    planes = layout("yuv422p16", w, h)
    p = synth.base_kernel_params(w, h, pixel_type="Luma16", lens="opencv_fisheye", digital_lens="gopro_superview")
    org, sm = synth.synthetic_gyro(2.0)
    cp = g.ComputeParams(p, org, sm)
    st = g.stab_config(p, "Luma16", digital_lens="gopro_superview")
    geo = [(pw, ph, pw * 2) for _, (pw, ph) in planes]
    srcs = [synth.synthetic_frame(pw, ph, "Luma16", frame=i, stride=s) for i, (pw, ph, s) in enumerate(geo)]
    tsrc = [torch.from_numpy(a).cuda() for a in srcs]
    outs = [torch.zeros(ph * s, dtype=torch.uint8, device="cuda") for pw, ph, s in geo]
    bufs = [g.Buffers(g.BufferDescription((pw, ph, s), a.data_ptr(), length=a.numel()), g.BufferDescription((pw, ph, s), o.data_ptr(), length=o.numel()))
            for (pw, ph, s), a, o in zip(geo, tsrc, outs)]
    specs = [pl.to_c() for pl, _ in planes]
    q = g.RenderQueue.for_planes(cp, st, "opencv_fisheye", "gopro_superview", specs, [b.input for b in bufs], [b.output for b in bufs],
                                 depth=1, checksum=True)
    ts = 500.0
    sums = q.render([0], lambda f: ts, lambda f: bufs)
    q.close()
    dg = g.DeviceGyro(cp)
    mats = torch.zeros((max(w, h), 14), dtype=torch.float32, device="cuda")
    kp0, rows, _, mfov = dg.frame_transform(ts, mats.data_ptr(), mats.shape[0], frame=0, with_fov=True)
    table = mats.cpu().numpy()[:rows].copy()
    dg.close()
    descs = []
    for i, (pl, _) in enumerate(planes):
        pw, ph, s = geo[i]
        stp = abi.StabConfig.from_buffer_copy(st)
        kp = kp0.copy()
        g.get_frame_transform_at(stp, cp, bufs[i], kp, frame=0, minimal_fov=mfov, timestamp_ms=ts)
        kp.pixel_value_limit = kp.max_pixel_value = pl.max_value
        kp.plane_index = i
        want = np.zeros(ph * s, np.uint8)
        assert oracle_lib.undistort_image(srcs[i], want, kp, "Luma16", "opencv_fisheye", "gopro_superview", table) == 0
        got = outs[i].cpu().numpy()
        assert checksum_host(got) == checksum_host(want), "plane %d" % i
        descs.append((want, s, s, ph))
    assert sums[0] == checksum_planes_host(descs)


# ---- two ranks: a sharded NV12 job, frame checksums gathered in frame order --------------------------------------------------------
N_FRAMES = 6
W2, H2 = 320, 180


def _nv12_job_rank(rank, world, dev_index, cdev, dist):
    """Rank `rank`'s frames of one NV12 job (DEVICE buffers) through a planes queue; returns {frame: checksum} gathered over the ranks."""
    import torch
    planes = layout("nv12", W2, H2)
    p = synth.base_kernel_params(W2, H2, pixel_type="Luma8")
    org, sm = cases.gyro()
    cp = g.ComputeParams(p, org, sm)
    st = g.stab_config(p, "Luma8")
    geo = [(pw, ph, pw * _bpp(pl.pixel_type)) for pl, (pw, ph) in planes]
    srcs = [torch.from_numpy(synth.synthetic_frame(pw, ph, pl.pixel_type, frame=i, stride=s)).cuda() for i, ((pl, _), (pw, ph, s)) in enumerate(zip(planes, geo))]
    mine = render_queue.shard_frames(N_FRAMES, world, rank)
    outs = {f: [torch.zeros(ph * s, dtype=torch.uint8, device="cuda") for pw, ph, s in geo] for f in mine}
    mk = lambda f: [g.Buffers(g.BufferDescription((pw, ph, s), a.data_ptr(), length=a.numel()), g.BufferDescription((pw, ph, s), o.data_ptr(), length=o.numel()))
                    for (pw, ph, s), a, o in zip(geo, srcs, outs[f])]
    specs = [pl.to_c() for pl, _ in planes]
    b0 = mk(mine[0])
    q = g.RenderQueue.for_planes(cp, st, "opencv_fisheye", None, specs, [b.input for b in b0], [b.output for b in b0], device=dev_index, depth=2, checksum=True)
    local = q.render(mine, lambda f: 250.0 + f * (1000.0 / FPS), mk)
    q.close()
    return render_queue.gather_results(local, dist, torch, cdev)


def _two_rank_worker(rank, world, port, n_gpus, outq):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev_index = rank % n_gpus
    torch.cuda.set_device(dev_index)
    if n_gpus >= world:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", dev_index))
        cdev = torch.device("cuda", dev_index)
    else:                                                      # one GPU: both ranks share it, the bookkeeping collective runs on gloo
        dist.init_process_group("gloo", rank=rank, world_size=world)
        cdev = torch.device("cpu")
    allr = _nv12_job_rank(rank, world, dev_index, cdev, dist)
    if rank == 0:
        outq.put((allr, dist.get_backend()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.fixture
def two_ranks():
    """Run _two_rank_worker on two processes (NCCL with two GPUs, gloo on one, as tests/test_render_queue.py does); returns rank 0's
    gathered result and the backend."""
    import torch
    import torch.multiprocessing as mp

    def run():
        n_gpus = torch.cuda.device_count()
        assert n_gpus >= 1
        s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
        ctx = mp.get_context("spawn")
        outq = ctx.Queue()
        procs = [ctx.Process(target=_two_rank_worker, args=(r, 2, port, n_gpus, outq)) for r in range(2)]
        for pr in procs: pr.start()
        got, backend = outq.get(timeout=300)
        for pr in procs:
            pr.join(timeout=120)
            assert pr.exitcode == 0
        assert backend == ("nccl" if n_gpus >= 2 else "gloo")
        return got
    return run


@pytest.mark.gpu
def test_two_ranks_render_a_sharded_nv12_job(two_ranks):
    import torch
    got = two_ranks()
    assert list(got) == list(range(N_FRAMES))
    planes = layout("nv12", W2, H2)
    p = synth.base_kernel_params(W2, H2, pixel_type="Luma8")
    org, sm = cases.gyro()
    cp = g.ComputeParams(p, org, sm)
    st = g.stab_config(p, "Luma8")
    dg = g.DeviceGyro(cp)
    mats = torch.zeros((max(W2, H2), 14), dtype=torch.float32, device="cuda")
    geo = [(pw, ph, pw * _bpp(pl.pixel_type)) for pl, (pw, ph) in planes]
    srcs = [synth.synthetic_frame(pw, ph, pl.pixel_type, frame=i, stride=s) for i, ((pl, _), (pw, ph, s)) in enumerate(zip(planes, geo))]
    for f in range(N_FRAMES):
        ts = 250.0 + f * (1000.0 / FPS)
        kp0, rows, _, mfov = dg.frame_transform(ts, mats.data_ptr(), mats.shape[0], frame=f, with_fov=True)
        table = mats.cpu().numpy()[:rows].copy()
        descs = []
        for i, (pl, _) in enumerate(planes):
            pw, ph, s = geo[i]
            stp = abi.StabConfig.from_buffer_copy(st); stp.pixel_type = abi.PIXEL_TYPES[pl.pixel_type][0]
            want = np.zeros(ph * s, np.uint8)
            bh = g.Buffers(g.BufferDescription((pw, ph, s), srcs[i]), g.BufferDescription((pw, ph, s), want))
            kp = kp0.copy()
            g.get_frame_transform_at(stp, cp, bh, kp, frame=f, minimal_fov=mfov, timestamp_ms=ts)
            kp.pixel_value_limit = kp.max_pixel_value = pl.max_value
            kp.plane_index = i
            assert oracle_lib.undistort_image(srcs[i], want, kp, pl.pixel_type, "opencv_fisheye", None, table) == 0
            descs.append((want, s, s, ph))
        assert got[f] == checksum_planes_host(descs), "frame %d rendered by rank %d" % (f, f % 2)
    dg.close()
