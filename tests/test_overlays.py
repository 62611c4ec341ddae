"""Preview overlays (SURVEY §8 f4, second half): draw_pixel + draw_safe_area of the reference's GPU kernels
(src/core/gpu/opencl_undistort.cl:109-154), off by default like the CPU path, on after gf_cuda_set_overlays.
Expected image = oracle restatement: stage-0 drawing entries onto the input, the CPU warp, stage-1 entries + safe-area shading onto
the output."""
import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi
from tests import cases, oracle_lib


def _drawing(p, scale, seed):
    """A canvas like gpu/drawing.rs builds: one byte per (x / scale, y / scale) cell = colour << 3 | alpha << 1 | stage."""
    rng = np.random.default_rng(seed)
    dw = max(p.width, p.output_width)
    cw, ch = int(dw / scale) + 2, int(max(p.height, p.output_height) / scale) + 2
    d = np.zeros(cw * ch, np.uint8)
    idx = rng.choice(d.size, d.size // 5, replace=False)
    d[idx] = (rng.integers(1, 11, idx.size) << 3 | rng.integers(0, 4, idx.size) << 1 | rng.integers(0, 2, idx.size)).astype(np.uint8)   # colours 9, 10 are ignored
    return d


def test_oracle_overlay_known_answers():
    p, src, m, mesh, dst0, pix, lens, digital = cases.build(dict(w=32, h=16, pix="RGBA8"))
    p.flags |= abi.FLAG_DRAWING_ENABLED; p.canvas_scale = 1.0
    buf = np.full((16, p.output_stride), 100, np.uint8)
    d = np.zeros(64 * 32, np.uint8)
    d[3 * 32 + 5] = (1 << 3) | (0 << 1) | 1            # red, alpha 1.0, output stage, at (x 5, y 3)
    d[4 * 32 + 6] = (2 << 3) | (2 << 1) | 0            # green, alpha 0.5, INPUT stage: ignored on the output
    p.safe_area_rect[:] = [4.0, 2.0, 27.0, 13.0]
    oracle_lib.draw_overlays(buf, 32, 16, p.output_stride, p, "RGBA8", False, d)
    px = lambda x, y: list(buf[y, x * 4:x * 4 + 4])
    assert px(5, 3) == [255, 0, 0, 255]
    assert px(6, 4) == [100, 100, 100, 100]
    assert px(1, 8) == [25, 25, 25, 100]               # outside the safe area, within its 5 px border: halved twice (alpha untouched)
    assert px(10, 8) == [100, 100, 100, 100]
    p.safe_area_rect[:] = [12.0, 6.0, 20.0, 10.0]
    buf[:] = 100
    oracle_lib.draw_overlays(buf, 32, 16, p.output_stride, p, "RGBA8", False, None)
    assert px(0, 0) == [50, 50, 50, 100] and px(8, 7) == [25, 25, 25, 100] and px(15, 8) == [100, 100, 100, 100]


@pytest.mark.gpu
@pytest.mark.parametrize("case,scale", [
    (dict(w=320, h=180), 1.0), (dict(w=320, h=180, pix="Luma16", lens="sony"), 2.0), (dict(w=203, h=117, pix="RGB8", stride_pad=3), 1.5),
    (dict(w=320, h=180, pix="RGBAf", interp="Lanczos4"), 1.0), (dict(w=320, h=180, ow=240, oh=136, pix="UV8"), 1.0),
])
def test_overlays_match_oracle(case, scale):
    import torch
    p, src, m, mesh, dst0, pix, lens, digital = cases.build(case)
    p.flags |= abi.FLAG_DRAWING_ENABLED; p.canvas_scale = scale
    ow, oh = p.output_width, p.output_height
    p.safe_area_rect[:] = [ow * 0.12, oh * 0.1, ow * 0.88, oh * 0.9]
    d = _drawing(p, scale, 3)
    # expected: input-stage entries onto a copy of the input, the CPU warp, output-stage entries + safe area onto the result
    src2 = src.copy()
    oracle_lib.draw_overlays(src2, case["w"], case["h"], p.stride, p, pix, True, d)
    assert not np.array_equal(src2, src)
    want = dst0.copy()
    assert oracle_lib.undistort_image(src2, want, p, pix, lens, digital, m, mesh) == 0
    oracle_lib.draw_overlays(want, ow, oh, p.output_stride, p, pix, False, d)
    itm = g.FrameTransform(matrices=m, kernel_params=p)
    for device_buffers in (False, True):
        got = dst0.copy()
        if device_buffers:
            tsrc, tdst = torch.from_numpy(src).cuda(), torch.from_numpy(got).cuda()
            bufs = g.Buffers(g.BufferDescription((case["w"], case["h"], p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                             g.BufferDescription((ow, oh, p.output_stride), tdst.data_ptr(), length=tdst.numel()))
        else:
            bufs = g.Buffers(g.BufferDescription((case["w"], case["h"], p.stride), src), g.BufferDescription((ow, oh, p.output_stride), got))
        w = g.CudaWrapper.new(p, pix, lens, digital, bufs)
        # off by default: identical to the CPU path, the drawing buffer is ignored
        plain = dst0.copy()
        assert oracle_lib.undistort_image(src, plain, p, pix, lens, digital, m, mesh) == 0
        w.undistort_image(bufs, itm, drawing_buffer=d); w.synchronize()
        if device_buffers: torch.cuda.synchronize(); got = tdst.cpu().numpy()
        assert np.array_equal(got, plain)
        w.set_overlays(True)
        if device_buffers: tdst.copy_(torch.from_numpy(dst0))
        else: got[:] = dst0
        w.undistort_image(bufs, itm, drawing_buffer=d); w.synchronize()
        if device_buffers:
            torch.cuda.synchronize(); got = tdst.cpu().numpy()
            assert np.array_equal(tsrc.cpu().numpy(), src)          # the caller's input buffer is never drawn into
        n = int((got != want).sum())
        assert n == 0, (n, device_buffers)
        w.close()


@pytest.mark.gpu
def test_host_planes_around_an_overlay_frame():
    """One HOST context renders the planes of a frame, then (overlays on) a frame whose drawing buffer makes the context allocate its
    drawing copies, then the planes again: growing the drawing buffers leaves the planes' staging buffers alone."""
    case = dict(w=320, h=180, pix="Luma16")
    built = [cases.build(dict(case, frame=i)) for i in range(2)]
    p0, src0, m, mesh, dst0, pix, lens, digital = built[0]
    mesh_data = mesh if mesh is not None else np.zeros(0, np.float32)
    params, wants = [], []
    for i, (p, src, _, _, d0, _, _, _) in enumerate(built):
        p = p.copy(); p.plane_index = i
        want = d0.copy()
        assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
        params.append(p); wants.append(want)

    def buffers(p, src, dst):
        return g.Buffers(g.BufferDescription((case["w"], case["h"], p.stride), src), g.BufferDescription((case["w"], case["h"], p.output_stride), dst))

    def planes():
        gots = [b[4].copy() for b in built]
        w.undistort_planes([buffers(p, b[1], got) for p, b, got in zip(params, built, gots)], params,
                           g.FrameTransform(matrices=m, kernel_params=params[0], mesh_data=mesh_data))
        for i, (got, want) in enumerate(zip(gots, wants)):
            assert np.array_equal(got, want), i

    # the overlay frame and its restatement: input-stage entries, the CPU warp, output-stage entries + safe area
    po = p0.copy()
    po.flags |= abi.FLAG_DRAWING_ENABLED; po.canvas_scale = 1.0
    po.safe_area_rect[:] = [case["w"] * 0.12, case["h"] * 0.1, case["w"] * 0.88, case["h"] * 0.9]
    d = _drawing(po, 1.0, 5)
    src2 = src0.copy()
    oracle_lib.draw_overlays(src2, case["w"], case["h"], po.stride, po, pix, True, d)
    want = dst0.copy()
    assert oracle_lib.undistort_image(src2, want, po, pix, lens, digital, m, mesh) == 0
    oracle_lib.draw_overlays(want, case["w"], case["h"], po.output_stride, po, pix, False, d)

    w = g.CudaWrapper.new(params[0], pix, lens, digital, buffers(params[0], src0, dst0.copy()))
    try:
        planes()
        w.set_overlays(True)
        got = dst0.copy()
        w.undistort_image(buffers(po, src0, got), g.FrameTransform(matrices=m, kernel_params=po, mesh_data=mesh_data), drawing_buffer=d)
        w.synchronize()
        assert np.array_equal(got, want)
        planes()
    finally:
        w.close()
