"""Shared case builder for the parity tests: one dict describes a warp call; `build` turns it into
(KernelParams, src, matrices, mesh) the way the reference's callers would (rendering/mod.rs:531-542)."""
import math

import numpy as np

from gyroflow_b200 import abi, synth
from tests import np_producer

_GYRO = {}


def gyro(duration=4.0):
    if duration not in _GYRO:
        _GYRO[duration] = synth.synthetic_gyro(duration)
    return _GYRO[duration]


def build(case):
    """case keys: w,h [,ow,oh] pix lens [digital] [interp] [rs] [ts] [stride_pad] [edge_values] [flags] [clear_flags] plus any KernelParams field override
    under 'params' and rects under 'in_rect'/'out_rect' (x,y,w,h) with 'in_size'/'out_size' = buffer (w,h)."""
    w, h = case["w"], case["h"]
    ow, oh = case.get("ow", w), case.get("oh", h)
    pix = case.get("pix", "RGBA8")
    lens = case.get("lens", "opencv_fisheye")
    digital = case.get("digital")
    _, count, sdt = abi.PIXEL_TYPES[pix]
    bpp = count * np.dtype(sdt).itemsize
    # buffers may be larger than the frame (planes with rects) and strides may be odd
    bw, bh = case.get("in_size", (w, h))
    obw, obh = case.get("out_size", (ow, oh))
    pad = case.get("stride_pad", 0)
    stride = bw * bpp + pad
    ostride = obw * bpp + case.get("out_stride_pad", pad)
    p = synth.base_kernel_params(w, h, ow, oh, pix, stride, ostride, lens, digital, case.get("interp", "Bilinear"), case.get("fov", 1.0))
    if case.get("edge_values"):      # content at the edges of the value domain (synth.edge_frame)
        src = synth.edge_frame(bw, bh, pix, seed=case.get("frame", 0), stride=stride)
    else:
        src = synth.synthetic_frame(bw, bh, pix, frame=case.get("frame", 0), stride=stride)
    if "in_rect" in case:
        p.source_rect[:] = list(case["in_rect"]); p.flags |= abi.FLAG_HAS_SOURCE_RECT
    else:
        p.source_rect[:] = [0, 0, bw, bh]
        if (bw, bh) != (w, h): p.flags |= abi.FLAG_HAS_SOURCE_RECT
    if "out_rect" in case:
        p.output_rect[:] = list(case["out_rect"]); p.flags |= abi.FLAG_HAS_OUTPUT_RECT
    else:
        p.output_rect[:] = [0, 0, obw, obh]
        if (obw, obh) != (ow, oh): p.flags |= abi.FLAG_HAS_OUTPUT_RECT
    for k, v in case.get("params", {}).items():
        cur = getattr(p, k)
        if hasattr(cur, "__len__"):
            cur[:] = list(v)
        else:
            setattr(p, k, v)
    if case.get("horizontal_rs"):
        p.flags |= abi.FLAG_HORIZONTAL_RS
    if case.get("flags"):
        p.flags |= case["flags"]
    if case.get("clear_flags"):
        p.flags &= ~case["clear_flags"]
    rs = case.get("rs", True)
    if case.get("identity"):
        m = np_producer.identity_matrices(p, rows=(h if rs else 1))
    else:
        org, sm = gyro()
        ibis = None
        if case.get("ibis"):
            n = p.width if case.get("horizontal_rs") else p.height
            def ibis(y, n=n):
                t = y / max(n - 1, 1)
                return (3.0 * math.sin(6.28 * t), -3.0 * math.cos(6.28 * t), math.radians(0.2) * math.sin(3.0 * t), math.sin(9.0 * t), -math.cos(5.0 * t))
        m = np_producer.frame_matrices(p, org, sm, case.get("ts", 1000.0), frame_readout_time_ms=(case.get("readout", 16.0) if rs else 0.0),
                                 video_rotation_deg=case.get("video_rotation", 0.0), horizontal=bool(case.get("horizontal_rs")), ibis=ibis)
    if case.get("matrix_hook"):
        m = np.ascontiguousarray(case["matrix_hook"](m.copy()), dtype=np.float32)
    p.matrix_count = m.shape[0]
    mesh = None
    if case.get("mesh"):
        mesh = synth.synthetic_mesh(w, h, n=case.get("mesh_n", 9), with_fpd=bool(case.get("fpd")))
    dst_init = np.full((obh, ostride), 0xA5, dtype=np.uint8)       # sentinel: untouched bytes must stay untouched
    return p, src, m, mesh, dst_init, pix, lens, digital


def compare(a, b, pix):
    """Return (n_mismatching_bytes, max_abs_diff) between two output buffers."""
    if a.shape != b.shape:
        return a.size, float("inf")
    diff = a != b
    n = int(diff.sum())
    if n == 0:
        return 0, 0.0
    _, count, sdt = abi.PIXEL_TYPES[pix]
    return n, float(np.abs(a.astype(np.int32) - b.astype(np.int32)).max())
