"""The warp context's one frame path: every gf_cuda_undistort_* entry point checks all of its arguments, in a fixed order, before it
enqueues anything; HOST frames and HOST planes go through the context's one staging; host tables are staged once per call."""
import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi
from tests import cases, oracle_lib

pytestmark = pytest.mark.gpu

BAD_PARAMS, SIZE_MISMATCH, BAD_STRIDE, UNSUPPORTED, TOO_SMALL, NO_DATA = -1, -3, -4, -5, -7, -8

# entry point -> (planes, tables on the device); DEVICE-table entry points get DEVICE buffers, the others HOST buffers
ENTRIES = {"image": (1, False), "image_async": (1, False), "image_dev": (1, True), "image_dev_flagged": (1, True),
           "planes_dev": (2, True), "planes_dev_flagged": (2, True), "planes": (2, False)}
SINGLE = ("image", "image_async", "image_dev", "image_dev_flagged")
PLANES_DEV = ("planes_dev", "planes_dev_flagged")


def _expect(single=None, planes_dev=None, planes=None, **by_entry):
    """(code, message fragment) per entry point; None: the fault does not apply to it."""
    e = {k: single for k in SINGLE}
    e.update({k: planes_dev for k in PLANES_DEV}, planes=planes)
    e.update(by_entry)
    return e


def _kind_fault(s, i):
    """Plane i's input of the kind its entry point refuses (a HOST plane where DEVICE ones are wanted and the other way round)."""
    s["ins"][i] = s["host_in"][i] if s["dev"] else s["dev_in"][i]


def _stride_fault(s, i):
    s["ps"][i].stride += 4                       # KernelParams stride differs from the buffer description


def _size_fault(s, i):
    s["ps"][i].width += 1                        # SizeMismatch against the context


def _long_host_input(s, i):
    s["ins"][i] = s["long_in"][i]                # longer than the context's HOST input (source_rect still inside it)


KIND = ("takes HOST", "takes DEVICE")
FAULTS = [
    # bad kind on plane 0 + bad stride on plane 1: the kind-then-validate loop runs plane by plane
    ("kind0_stride1", lambda s: (_kind_fault(s, 0), _stride_fault(s, 1)),
     _expect(planes_dev=(BAD_PARAMS, KIND[1]), planes=(BAD_PARAMS, KIND[0]))),
    ("stride0_kind1", lambda s: (_stride_fault(s, 0), _kind_fault(s, 1)),
     _expect(planes_dev=(BAD_STRIDE, "stride differs"), planes=(BAD_STRIDE, "stride differs"))),
    # one plane: a buffer of no kind is refused by validate after its stride checks
    ("nokind_stride", lambda s: (s["ins"][0].__setattr__("kind", abi.BUF_NONE), _stride_fault(s, 0)),
     _expect(single=(BAD_STRIDE, "stride differs"))),
    # every plane's validate runs before the first plane's checks against the context
    ("size0_stride1", lambda s: (_size_fault(s, 0), _stride_fault(s, 1)),
     _expect(planes_dev=(BAD_STRIDE, "stride differs"), planes=(BAD_STRIDE, "stride differs"))),
    ("size0_kind1", lambda s: (_size_fault(s, 0), _kind_fault(s, 1)),
     _expect(planes_dev=(BAD_PARAMS, KIND[1]), planes=(BAD_PARAMS, KIND[0]))),
    ("null_matrices_oversize_mesh", lambda s: s.update(mats=None, mesh_len=840),
     _expect(single=(NO_DATA, "NoStabilizationData"), planes_dev=(NO_DATA, "NoStabilizationData"), planes=(NO_DATA, "NoStabilizationData"))),
    # SizeMismatch + a HOST input beyond the context's staging (gf_cuda_undistort_planes grows its staging; the DEVICE form refuses HOST)
    ("size_long_host", lambda s: ([_size_fault(s, i) for i in range(len(s["ps"]))], _long_host_input(s, 0)),
     _expect(single=(SIZE_MISMATCH, "SizeMismatch"), planes_dev=(BAD_PARAMS, KIND[1]), planes=(SIZE_MISMATCH, "SizeMismatch"))),
    ("long_host_input", lambda s: _long_host_input(s, 0),
     _expect(single=(TOO_SMALL, "Buffer size mismatch input"), planes_dev=(BAD_PARAMS, KIND[1]))),
    ("long_host_output", lambda s: s["outs"].__setitem__(0, s["long_out"][0]),
     _expect(single=(TOO_SMALL, "Buffer size mismatch output"), planes_dev=(BAD_PARAMS, KIND[1]))),
    ("long_host_input_and_output", lambda s: (_long_host_input(s, 0), s["outs"].__setitem__(0, s["long_out"][0])),
     _expect(single=(TOO_SMALL, "Buffer size mismatch input"), planes_dev=(BAD_PARAMS, KIND[1]))),
    # misaligned device table + a mesh shorter than its header: the mesh checks come first (host tables have no alignment check)
    ("misaligned_table_short_mesh", lambda s: s.update(mats=s["mats"] + 4, mesh_len=5),
     _expect(single=(BAD_PARAMS, "mesh shorter"), planes_dev=(BAD_PARAMS, "mesh shorter"), planes=(BAD_PARAMS, "mesh shorter"))),
    ("misaligned_table", lambda s: s.update(mats=s["mats"] + 4),
     _expect(image_dev=(BAD_PARAMS, "8-byte aligned"), image_dev_flagged=(BAD_PARAMS, "8-byte aligned"), planes_dev=(BAD_PARAMS, "8-byte aligned"))),
    ("interpolation_short_table", lambda s: ([p.__setattr__("interpolation", abi.INTERP["Bicubic"]) for p in s["ps"]], s.update(rows=s["rows"] - 1)),
     _expect(single=(UNSUPPORTED, "interpolation"), planes_dev=(UNSUPPORTED, "interpolation"), planes=(UNSUPPORTED, "interpolation"))),
    ("short_table_null_mesh", lambda s: s.update(rows=s["rows"] - 1, mesh=None, mesh_len=9),
     _expect(single=(TOO_SMALL, "matrix_count > rows"), planes_dev=(TOO_SMALL, "matrix_count > rows"), planes=(TOO_SMALL, "matrix_count > rows"))),
    ("null_mesh_short_mesh_pointer", lambda s: s.update(mesh=None, mesh_len=5),
     _expect(single=(BAD_PARAMS, "mesh is null"), planes_dev=(BAD_PARAMS, "mesh is null"), planes=(BAD_PARAMS, "mesh is null"))),
    # host tables with more rows than the context holds + a HOST input beyond staging: the table check comes first
    ("long_host_table_long_host", lambda s: (s.update(rows=65) if not s["tables_dev"] else None, _long_host_input(s, 0)),
     _expect(image=(TOO_SMALL, "Buffer size mismatch matrices"), image_async=(TOO_SMALL, "Buffer size mismatch matrices"),
             image_dev=(TOO_SMALL, "Buffer size mismatch input"), image_dev_flagged=(TOO_SMALL, "Buffer size mismatch input"),
             planes_dev=(BAD_PARAMS, KIND[1]), planes=(TOO_SMALL, "Buffer size mismatch matrices"))),
]


def _call(w, entry, s, stream=None):
    lib, h = w._lib, w._h
    n = len(s["ps"])
    ins, outs, ps = (abi.BufferDesc * n)(*s["ins"]), (abi.BufferDesc * n)(*s["outs"]), (abi.KernelParams * n)(*s["ps"])
    mats, rows, mesh, mesh_len, flags = s["mats"], s["rows"], s["mesh"], s["mesh_len"], s["flags"]
    if entry == "image":
        return lib.gf_cuda_undistort_image(h, ins, outs, ps, mats, rows, mesh, mesh_len, None, 0, stream)
    if entry == "image_async":
        return lib.gf_cuda_undistort_image_async(h, ins, outs, ps, mats, rows, mesh, mesh_len, stream)
    if entry == "image_dev":
        return lib.gf_cuda_undistort_image_dev(h, ins, outs, ps, mats, rows, mesh, mesh_len, stream)
    if entry == "image_dev_flagged":
        return lib.gf_cuda_undistort_image_dev_flagged(h, ins, outs, ps, mats, rows, mesh, mesh_len, flags, stream)
    if entry == "planes_dev":
        return lib.gf_cuda_undistort_planes_dev(h, n, ins, outs, ps, mats, rows, mesh, mesh_len, stream)
    if entry == "planes_dev_flagged":
        return lib.gf_cuda_undistort_planes_dev_flagged(h, n, ins, outs, ps, mats, rows, mesh, mesh_len, flags, stream)
    return lib.gf_cuda_undistort_planes(h, n, ins, outs, ps, mats, rows, mesh, mesh_len, stream)


def test_check_order_per_entry_point():
    """Jobs with two faults each, through each of the seven entry points: the code (and the reason) of the check that comes first, and
    nothing enqueued — HOST outputs untouched, no launch counted."""
    import torch
    built = [cases.build(dict(w=64, h=36, frame=i)) for i in range(2)]
    p0, _, m, _, _, pix, lens, digital = built[0]
    mesh = np.zeros(840, np.float32)
    tm, tmesh = torch.from_numpy(m).cuda(), torch.from_numpy(mesh).cuda()
    tflags = torch.zeros(1, dtype=torch.int32, device="cuda")
    keep = []                                    # every buffer a description points to outlives the calls

    def host(arr, stride):
        keep.append(arr)
        return g.BufferDescription((64, 36, stride), arr).to_c()

    def dev(arr, stride):
        t = torch.from_numpy(arr).cuda()
        keep.append(t)
        return g.BufferDescription((64, 36, stride), t.data_ptr(), length=t.numel()).to_c()

    w = g.CudaWrapper.new(p0, pix, lens, digital, g.Buffers(g.BufferDescription((64, 36, p0.stride), built[0][1]),
                                                              g.BufferDescription((64, 36, p0.output_stride), built[0][4].copy())))
    torch.cuda.synchronize()
    try:
        for entry, (n, tables_dev) in ENTRIES.items():
            for name, fault, expected in FAULTS:
                if expected[entry] is None:
                    continue
                srcs = [b[1] for b in built[:n]]
                host_outs = [b[4].copy() for b in built[:n]]
                long_outs = [np.full((40, p0.output_stride), 0xA5, np.uint8) for _ in range(n)]
                s = dict(dev=tables_dev, tables_dev=tables_dev, ps=[], ins=[], outs=[],
                         host_in=[host(a, p0.stride) for a in srcs], dev_in=[dev(a, p0.stride) for a in srcs],
                         long_in=[host(np.concatenate([a, np.zeros((4, p0.stride), np.uint8)]), p0.stride) for a in srcs],
                         long_out=[host(a, p0.output_stride) for a in long_outs],
                         mats=tm.data_ptr() if tables_dev else m.ctypes.data, rows=m.shape[0],
                         mesh=tmesh.data_ptr() if tables_dev else mesh.ctypes.data, mesh_len=0, flags=tflags.data_ptr())
                for i in range(n):
                    p = built[i][0].copy(); p.plane_index = i
                    s["ps"].append(p)
                    s["ins"].append(s["dev_in"][i] if tables_dev else s["host_in"][i])
                    s["outs"].append(dev(built[i][4], p0.output_stride) if tables_dev else host(host_outs[i], p0.output_stride))
                fault(s)
                l0 = w.launch_count
                rc = _call(w, entry, s)
                msg = (w._lib.gf_cuda_last_error(w._h) or b"").decode()
                w.synchronize(); torch.cuda.synchronize()
                code, fragment = expected[entry]
                assert rc == code, (entry, name, rc, msg)
                assert fragment in msg, (entry, name, msg)
                assert w.launch_count == l0, (entry, name)
                for i in range(n):
                    assert np.array_equal(host_outs[i], built[i][4]) and (long_outs[i] == 0xA5).all(), (entry, name, i)
    finally:
        w.close()


def _oracle(p, src, dst0, pix, lens, digital, m, mesh):
    want = dst0.copy()
    assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
    return want


def test_host_planes_not_fused_between_single_plane_calls():
    """One HOST context with host tables and a mesh: a frame, then three planes that do not fuse (their lens_correction_amount differs)
    in buffers larger than the context's (its staging grows), then the frame again.  Every output equals the oracle, each call counts
    the launches it always has, and the single-plane call still refuses the larger buffers."""
    case = dict(w=320, h=180, mesh=True)
    p, src, m, mesh, dst0, pix, lens, digital = cases.build(case)
    itm = g.FrameTransform(matrices=m, kernel_params=p, mesh_data=mesh)
    big = dict(case, in_size=(400, 200), in_rect=(40, 10, 320, 180), out_size=(352, 200), out_rect=(16, 10, 320, 180))
    planes = [cases.build(dict(big, frame=i + 1, params=dict(lens_correction_amount=amount))) for i, amount in enumerate((1.0, 0.6, 0.35))]
    params = []
    for i, b in enumerate(planes):
        q = b[0].copy(); q.plane_index = i
        params.append(q)
    wants = [_oracle(q, b[1], b[4], pix, lens, digital, m, mesh) for q, b in zip(params, planes)]
    want = _oracle(p, src, dst0, pix, lens, digital, m, mesh)

    def frame():
        got = dst0.copy()
        l0 = w.launch_count
        w.undistort_image(g.Buffers(g.BufferDescription((320, 180, p.stride), src), g.BufferDescription((320, 180, p.output_stride), got)), itm)
        assert w.launch_count - l0 == 1                   # a mesh: the general kernel, one launch
        assert np.array_equal(got, want)

    w = g.CudaWrapper.new(p, pix, lens, digital, g.Buffers(g.BufferDescription((320, 180, p.stride), src),
                                                             g.BufferDescription((320, 180, p.output_stride), dst0.copy())))
    try:
        frame()
        gots = [b[4].copy() for b in planes]
        bufs = [g.Buffers(g.BufferDescription((400, 200, q.stride), b[1]), g.BufferDescription((352, 200, q.output_stride), got))
                for q, b, got in zip(params, planes, gots)]
        l0 = w.launch_count
        w.undistort_planes(bufs, params, g.FrameTransform(matrices=m, kernel_params=params[0], mesh_data=mesh))
        assert w.launch_count - l0 == len(planes)          # not fused: every plane on its own, one launch each
        for i, (got, wp) in enumerate(zip(gots, wants)):
            assert np.array_equal(got, wp), i
        frame()
        with pytest.raises(g.GyroflowCoreError) as e:
            w.undistort_image(bufs[0], g.FrameTransform(matrices=m, kernel_params=params[0], mesh_data=mesh))
        assert e.value.kind == "BufferTooSmall"
        frame()
    finally:
        w.close()


def test_async_host_calls_on_two_streams():
    """Two gf_cuda_undistort_image_async calls with HOST buffers on one context, on two streams, with no wait in between: both stage
    through the same device buffers (the outputs are not covered by the warp, so each is uploaded and copied back whole), and the
    second waits for the first on the device."""
    import torch
    case = dict(w=320, h=180, out_size=(352, 200), out_rect=(16, 10, 320, 180))
    frames = [cases.build(dict(case, frame=i)) for i in range(2)]
    p, _, m, mesh, _, pix, lens, digital = frames[0]
    wants = [_oracle(f[0], f[1], f[4], pix, lens, digital, f[2], f[3]) for f in frames]
    srcs = [f[1].copy() for f in frames]
    gots = [f[4].copy() for f in frames]
    for a in srcs + gots:
        g.host_register(a)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    w = g.CudaWrapper.new(p, pix, lens, digital, g.Buffers(g.BufferDescription((320, 180, p.stride), srcs[0]),
                                                             g.BufferDescription((352, 200, p.output_stride), gots[0])))
    try:
        for f, s, got, st in zip(frames, srcs, gots, streams):
            bufs = g.Buffers(g.BufferDescription((320, 180, f[0].stride), s), g.BufferDescription((352, 200, f[0].output_stride), got))
            w.undistort_image_async(bufs, g.FrameTransform(matrices=f[2], kernel_params=f[0]), stream=st.cuda_stream)
        w.synchronize()
        for i, (got, want) in enumerate(zip(gots, wants)):
            assert np.array_equal(got, want), i
    finally:
        w.close()
        for a in srcs + gots:
            g.host_unregister(a)


def test_mixed_buffer_kinds():
    """gf_cuda_undistort_image with a HOST input and a DEVICE output, and with a DEVICE input and a HOST output whose stride is padded
    and whose output rect leaves a border: the pixels match the oracle, and the padding and border keep their bytes."""
    import torch
    case = dict(w=320, h=180, stride_pad=12, out_size=(352, 200), out_rect=(16, 10, 320, 180))
    p, src, m, mesh, dst0, pix, lens, digital = cases.build(case)
    want = _oracle(p, src, dst0, pix, lens, digital, m, mesh)
    itm = g.FrameTransform(matrices=m, kernel_params=p)
    host_in, host_out = g.BufferDescription((320, 180, p.stride), src), g.BufferDescription((352, 200, p.output_stride), dst0.copy())
    w = g.CudaWrapper.new(p, pix, lens, digital, g.Buffers(host_in, host_out))
    try:
        tdst = torch.from_numpy(dst0).cuda()
        w.undistort_image(g.Buffers(host_in, g.BufferDescription((352, 200, p.output_stride), tdst.data_ptr(), length=tdst.numel())), itm)
        w.synchronize(); torch.cuda.synchronize()
        assert np.array_equal(tdst.cpu().numpy(), want)
        tsrc = torch.from_numpy(src).cuda()
        got = dst0.copy()
        torch.cuda.synchronize()
        w.undistort_image(g.Buffers(g.BufferDescription((320, 180, p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                                    g.BufferDescription((352, 200, p.output_stride), got)), itm)
        assert np.array_equal(got, want)
        assert (got[:, 352 * 4:] == 0xA5).all() and (got[:10] == 0xA5).all()      # padding and border as they were
    finally:
        w.close()
