"""EWA CubicBC resampling against the CPU oracle where the kernel matrix cannot reach.

test_kernel_matrix renders EWA in its two coordinate variants on every pair and pixel type; this file covers what a matrix cell
cannot express, byte for byte against oracle_lib.undistort_image:

  the footprint guard   a box of more than 2^22 taps is rendered as background, min(bg, pixel_value_limit) (sample_ewa in
                        csrc/warp_kernel.cuh), pixels on both sides of the threshold in one frame
  box_in                the fast path that skips the per-tap source-rect tests: boxes on each edge of a source rect inside a larger
                        input, and boxes one tap past each edge whose edge taps carry weight
  unaligned sources     F_SRC_VEC clear, so the taps go through load_bytes, in every pixel type
  fused planes          one coordinate pass with both probe maps shared by 2-4 planes with their own backgrounds

The one matrix cell EWA cannot be compared in (geometry B of opencv_fisheye + gopro_hyperview: NaN centres next to footprints past
the guard) is classified on the host; its NaN-centre pixels, the 0 / 0 path, are rendered on the GPU and compared with the value the
reference gives them, pixel_value_limit, since the oracle cannot finish that frame.

Where a test claims a class of footprints, the class is computed on the host the way the reference computes the footprint
(cpu_undistort.rs:565-572 and :331-335): the centre and both probes from oracle_lib.undistort_coord, None probes as (0, 0), the box
from np_restatement.affine_bbox with Rust's saturating `as i32`; every class a test claims must be non-empty.
"""
import time

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi
from tests import cases, np_restatement, oracle_lib
from tests.test_kernel_matrix import GUARD, MODES, PIXEL_TYPES, _bpp_align, build, descs, geometries, render, report, set_switch

F = np.float32
EPS = F(0.01)
GUARD_TAPS = 1 << 22
EWA_MODES = [m for m in MODES if m[2].startswith("EWA")]


def footprint(p, m, lens, digital, x, y):
    """(centre, jac, box) of output buffer pixel (x, y): box = (b0, b1, b2, b3), the inclusive tap bounds.  (None, None, None) where
    the centre is None."""
    c = oracle_lib.undistort_coord(F(x), F(y), p, m, lens, digital)
    if c is None:
        return None, None, None
    u, v = c
    rx = oracle_lib.undistort_coord(F(x) + EPS, F(y), p, m, lens, digital) or (F(0.0), F(0.0))
    ry = oracle_lib.undistort_coord(F(x), F(y) + EPS, p, m, lens, digital) or (F(0.0), F(0.0))
    with np.errstate(invalid="ignore"):                               # NaN centres
        jac = ((rx[0] - u) / EPS, (ry[0] - u) / EPS, (rx[1] - v) / EPS, (ry[1] - v) / EPS)
        tx, ty = np_restatement.affine_bbox(jac)
        box = tuple(np_restatement.as_i32(f(w)) for f, w in ((np.floor, u - tx), (np.ceil, u + tx), (np.floor, v - ty), (np.ceil, v + ty)))
    return c, jac, box


def taps(box):
    b0, b1, b2, b3 = box
    return (b1 - b0 + 1) * (b3 - b2 + 1)


def edge_weighted(p, centre, jac, box, edge):
    """Does a tap on the box's edge `edge` (0: column b0, 1: column b1, 2: row b2, 3: row b3) have a non-zero filter weight?  The
    weights as sample_ewa computes them (cpu_undistort.rs:345-356): a tap whose weight is zero is never read."""
    u, v = centre
    A, B, Cc = np_restatement.clamped_ellipse(jac)
    b0, b1, b2, b3 = box
    line = [(box[edge], y) for y in range(b2, b3 + 1)] if edge < 2 else [(x, box[edge]) for x in range(b0, b1 + 1)]
    for x, y in line:
        fx, fy = F(x) - u, F(y) - v
        if np_restatement.bc2(np_restatement.sqrtf(fx * fx * A + fx * (fy * B) + fy * fy * Cc), p) != 0:
            return True
    return False


def rect_classes(p, centre, jac, box):
    """The source-rect classes of a footprint: ("edge", i) for a box inside the rect (the box_in fast path) that touches edge i of the
    rect, ("out", i) for a box one tap past edge i and inside the other three, with a non-zero weight on that edge's taps."""
    rx0, ry0 = p.source_rect[0], p.source_rect[1]
    rx1, ry1 = rx0 + p.source_rect[2], ry0 + p.source_rect[3]
    b0, b1, b2, b3 = box
    inside = (b0 >= rx0, b1 < rx1, b2 >= ry0, b3 < ry1)
    out = set()
    for i, (at, past) in enumerate(((b0 == rx0, b0 == rx0 - 1), (b1 == rx1 - 1, b1 == rx1), (b2 == ry0, b2 == ry0 - 1), (b3 == ry1 - 1, b3 == ry1))):
        others = all(inside[j] for j in range(4) if j != i)
        if at and all(inside):
            out.add(("edge", i))
        if past and others and edge_weighted(p, centre, jac, box, i):
            out.add(("out", i))
    return out


def written_pixels(case, pix, lens, digital, interp, out_len):
    """[(x, y)] of the output pixels the oracle writes (a byte it leaves alone keeps its fill, which differs between two runs)."""
    p, src, m, dst = build(case, pix, lens, digital, interp, out_len)
    runs = []
    for fill in (0xA5, 0x5A):
        out = np.full(out_len, fill, np.uint8)
        assert oracle_lib.undistort_image(src, out, p, pix, lens, digital, m) == 0
        runs.append(out)
    same = runs[0] == runs[1]
    bpp, _ = _bpp_align(pix)
    out = []
    for y in range(-(-out_len // p.output_stride)):
        for x in range(p.output_stride // bpp):
            off = y * p.output_stride + x * bpp
            if off + bpp <= out_len and same[off:off + bpp].all():
                out.append((x, y))
    return p, m, out


def _fisheye_case(**kw):
    return dict(dict(w=75, h=43, fov=1.3, lens="opencv_fisheye"), **kw)


def _is_nan(centre):
    return np.isnan(centre[0]) or np.isnan(centre[1])


def _render(case, pix, mode, out_len, kinds, code=None):
    """render() of test_kernel_matrix in one EWA variant: the plan code the variant names (or `code`), three coordinate passes and a
    sampling pass, no byte written past the output."""
    _, _, interp, tables, mode_code = mode
    code = mode_code if code is None else code
    want, outs, got = render(case, pix, case.get("lens", "opencv_fisheye"), case.get("digital"), interp, tables, out_len, kinds)
    assert got == code, (pix, mode[0], got, code)
    for kind, out, launches in outs:
        assert launches == 4, (pix, kind, launches)
        assert np.array_equal(out[out_len:], np.full(GUARD, 0xA5, np.uint8)), (pix, kind, "wrote past the end of the output")
    return want, outs


# ---- host classification, without a GPU ------------------------------------------------------------------------------------------
def test_geometry_b_footprints():
    """Geometry B of the kernel matrix for (opencv_fisheye, gopro_hyperview) has written pixels whose centre is NaN (the 0 / 0 path of
    sample_ewa), and next to them footprints past the 2^22-tap guard, which is why the matrix leaves that cell out of its EWA
    variants (EWA_UNCOMPARABLE).  Every other pair's geometry A and B footprints stay small, so the rest of the matrix compares
    byte for byte."""
    from tests.test_kernel_matrix import EWA_UNCOMPARABLE, library_pairs
    counts = {}
    for lens, digital in library_pairs():
        for gname, case, out_len in geometries("RGBA8"):
            if gname not in ("A/stride8", "B/ends-at-last-pixel"):
                continue
            p, m, written = written_pixels(case, "RGBA8", lens, digital, "Bilinear", out_len)
            nan, big = 0, 0
            for x, y in written:
                c, _, box = footprint(p, m, lens, digital, x, y)
                if c is not None and _is_nan(c):
                    nan += 1
                elif c is not None and taps(box) > 1000:
                    big = max(big, taps(box))
            counts[(lens, digital, gname[0])] = (nan, big)
    bad = {k for k, (nan, big) in counts.items() if nan or big}
    assert bad == EWA_UNCOMPARABLE, {k: counts[k] for k in bad}
    nan, big = counts[("opencv_fisheye", "gopro_hyperview", "B")]
    assert nan > 0 and big > GUARD_TAPS, (nan, big)


# box_in: a fisheye frame rolled by 45 degrees, with an output rect 12 pixels wide and 256 high standing for the 32 x 32 output.  The
# footprints are sheared ellipses, minified about 2.7x along one axis and magnified about 8x along the other; the ellipse clamped to
# at least one tap then reaches past affine_bbox's edge taps, so a box one tap past the rect has weighted taps outside it (with a
# round footprint those taps weigh 0 and are never read).  The source rect sits inside a larger input whose border holds other
# content than the background.
BOX_IN_CASE = dict(w=32, h=32, rs=False, video_rotation=-45.0, in_size=(44, 42), in_rect=(6, 5, 32, 32), out_size=(16, 260), out_rect=(2, 2, 12, 256))
BOX_IN_SHIFTS = [float(s) for s in np.arange(-2.0, 2.0, 0.25)]        # translation2d (s, 0.37 s): sub-pixel steps across every edge


def _box_in_case(s):
    return dict(BOX_IN_CASE, params=dict(translation2d=[s, 0.37 * s], background=[0.25, 0.5, 0.75, 1.0]))


def test_box_in_classes():
    """Over the translation sweep, written footprints fall in every class of rect_classes: boxes inside the rect touching each of its
    four edges (the fast path), and boxes one tap past each edge, inside the other three, with weighted taps on that edge."""
    classes = {}
    for s in BOX_IN_SHIFTS:
        p, _, m, _, _, _, lens, _ = cases.build(dict(_box_in_case(s), pix="RGBA8", lens="opencv_fisheye", interp="EWA: Robidoux"))
        ox, oy, ow, oh = list(p.output_rect)
        for y in range(oy, oy + oh):
            for x in range(ox, ox + ow):
                c, jac, box = footprint(p, m, lens, None, x, y)
                if c is not None and not _is_nan(c):
                    for k in rect_classes(p, c, jac, box):
                        classes[k] = classes.get(k, 0) + 1
    missing = [(kind, i) for kind in ("edge", "out") for i in range(4) if not classes.get((kind, i))]
    assert not missing, (missing, classes)


# ---- the GPU tests ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_box_in_boundary(request, monkeypatch):
    """The box_in sweep (test_box_in_classes) in every pixel type and both EWA variants, byte for byte against the oracle."""
    t0, n = time.perf_counter(), 0
    for pix in PIXEL_TYPES:
        for s in BOX_IN_SHIFTS:
            case = dict(_box_in_case(s), lens="opencv_fisheye")
            out_len = cases.build(dict(case, pix=pix))[4].size
            for mode in EWA_MODES:
                set_switch(monkeypatch, mode[1])
                want, outs = _render(case, pix, mode, out_len, ("host",))
                got = outs[0][1][:out_len]
                assert np.array_equal(got, want), (pix, s, mode[0], int((got != want).sum()))
                n += 1
    report(request, "test_box_in_boundary: %d renders (13 pixel types x %d shifts x 2 variants), %.1f s" % (n, len(BOX_IN_SHIFTS), time.perf_counter() - t0))
    assert n == 13 * len(BOX_IN_SHIFTS) * 2


@pytest.mark.gpu
@pytest.mark.parametrize("pix", ["Luma8", "Luma16"])
def test_footprint_guard(request, monkeypatch, pix):
    """A pure-minification 4096 x 4096 frame (the lens's "all coefficients zero" early-out, no rolling shutter) onto 8 x 6 pixels:
    about 512 source pixels per output pixel, so the boxes are about 2048 taps on a side.  Pixels whose box is over 2^22 taps are
    min(bg, pixel_value_limit) converted to the format (the background is the format's maximum, the limit 0.8 of it, so the min
    bites); every other pixel is the oracle's sum of its ~4M taps, below the limit."""
    set_switch(monkeypatch, None)
    t0 = time.perf_counter()
    _, _, sdt = abi.PIXEL_TYPES[pix]
    limit = {"u1": 204.0, "u2": 52428.0}[sdt]
    case = dict(w=4096, h=4096, ow=8, oh=6, fov=0.9992, identity=True, rs=False,
                params=dict(k=[0.0] * 12, background=[1.0, 1.0, 1.0, 1.0], pixel_value_limit=limit))
    mode = ("general-ewa", None, "EWA: Mitchell", "host", 0x10)             # pixel_value_limit is a general-only feature
    p, src, m, mesh, dst0, _, lens, digital = cases.build(dict(case, pix=pix, interp=mode[2]))
    bpp, _ = _bpp_align(pix)
    counts = np.array([[taps(footprint(p, m, lens, None, x, y)[2]) for x in range(8)] for y in range(6)])
    over = counts > GUARD_TAPS
    assert over.any() and not over.all(), counts
    below, above = int(counts[~over].max()), int(counts[over].min())
    out_len = dst0.size
    want, outs = _render(case, pix, mode, out_len, ("host",))
    bg = np.array([limit], dtype=sdt).view(np.uint8)
    assert not np.array_equal(bg, np.array([p.max_pixel_value], dtype=sdt).view(np.uint8))
    expect = want.copy()
    for y, x in zip(*np.nonzero(over)):
        off = y * p.output_stride + x * bpp
        assert not np.array_equal(want[off:off + bpp], bg), (x, y)           # the oracle's sum is not the background
        expect[off:off + bpp] = bg
    got = outs[0][1][:out_len]
    report(request, "test_footprint_guard[%s]: %d pixels over 2^22 taps, %d under; closest counts 2^22 - %d and 2^22 + %d; %.1f s" %
           (pix, int(over.sum()), int((~over).sum()), GUARD_TAPS - below, above - GUARD_TAPS, time.perf_counter() - t0))
    assert np.array_equal(got, expect), "%d bytes differ" % int((got != expect).sum())


@pytest.mark.gpu
def test_nan_centres(request, monkeypatch):
    """Geometry B of (opencv_fisheye, gopro_hyperview), which the matrix cannot compare: every written pixel whose centre is NaN has a
    1 x 1 box whose one tap has weight 0, so the reference divides 0 by 0 and f32::min turns the NaN into pixel_value_limit.  Every
    pixel type, both EWA variants, HOST buffers; the other pixels are not compared (the oracle cannot finish their footprints)."""
    from gyroflow_b200.abi import FLAG_FILL_WITH_BACKGROUND
    lens, digital = "opencv_fisheye", "gopro_hyperview"
    t0, n, n_nan = time.perf_counter(), 0, 0
    for pix in PIXEL_TYPES:
        bpp, _ = _bpp_align(pix)
        [(_, case, out_len)] = [gm for gm in geometries(pix) if gm[0] == "B/ends-at-last-pixel"]
        p, m, written = written_pixels(case, pix, lens, digital, "Bilinear", out_len)
        nan = [(x, y) for x, y in written if (lambda c: c is not None and _is_nan(c))(footprint(p, m, lens, digital, x, y)[0])]
        assert nan, pix
        # the limit in the format: the oracle's fill-with-background render with the background at the limit
        lim = dict(case, flags=FLAG_FILL_WITH_BACKGROUND, params=dict(background=[p.pixel_value_limit / p.max_pixel_value] * 4))
        lp, lsrc, lm, ldst = build(lim, pix, lens, digital, "Bilinear", out_len)
        want = ldst[:out_len].copy()
        assert oracle_lib.undistort_image(lsrc, want, lp, pix, lens, digital, lm) == 0
        for mode in EWA_MODES:
            set_switch(monkeypatch, mode[1])
            mp, src, mm, dst = build(case, pix, lens, digital, mode[2], out_len)
            bufs = descs(case, mp, src, dst, out_len)
            ctx = g.CudaWrapper.new(mp, pix, lens, digital, bufs)
            try:
                l0 = ctx.launch_count
                ctx.undistort_image(bufs, g.FrameTransform(matrices=mm, kernel_params=mp))
                ctx.synchronize()
                assert ctx.launch_count - l0 == 4
            finally:
                ctx.close()
            assert np.array_equal(dst[out_len:], np.full(GUARD, 0xA5, np.uint8)), (pix, mode[0])
            for x, y in nan:
                off = y * mp.output_stride + x * bpp
                assert np.array_equal(dst[off:off + bpp], want[off:off + bpp]), (pix, mode[0], (x, y), dst[off:off + bpp], want[off:off + bpp])
            n += 1
        n_nan += len(nan)
    report(request, "test_nan_centres: %d renders, %d NaN-centre pixels over the 13 pixel types, %.1f s" % (n, n_nan, time.perf_counter() - t0))
    assert n == 13 * 2


@pytest.mark.gpu
def test_unaligned_sources(request, monkeypatch):
    """EWA in every pixel type from a source the kernel may not read with whole-pixel vector loads: HOST with a stride one byte past an
    aligned one, DEVICE with the input pointer one byte past an aligned one.  For every layout whose pixels need more than byte
    alignment the feature word has F_SRC_VEC clear, so every tap goes through load_bytes."""
    from tests.test_feature_matrix import features
    t0, n = time.perf_counter(), 0
    for pix in PIXEL_TYPES:
        bpp, align = _bpp_align(pix)
        for kind, case in (("host", _fisheye_case(stride_pad=1)), ("device", _fisheye_case(stride_pad=align, src_offset=1))):
            out_len = 43 * (75 * bpp + case["stride_pad"])
            for mode in EWA_MODES:
                set_switch(monkeypatch, mode[1])
                _, word = features(case, pix, "opencv_fisheye", None, mode[2], out_len, "host")
                assert bool(word & abi.F["F_SRC_VEC"]) == (align == 1), (pix, kind, hex(word))
                # unaligned pixel access is general-only: both variants take the general coordinate pass then
                want, outs = _render(case, pix, mode, out_len, (kind,), code=mode[4] if align == 1 else 0x10)
                got = outs[0][1][:out_len]
                assert np.array_equal(got, want), (pix, kind, mode[0], int((got != want).sum()))
                n += 1
    report(request, "test_unaligned_sources: %d renders, %.1f s" % (n, time.perf_counter() - t0))
    assert n == 13 * 2 * 2


@pytest.mark.gpu
@pytest.mark.parametrize("pix,n_planes", [("Luma8", 3), ("Luma16", 2), ("UV8", 2), ("UV16", 3), ("R32f", 4)])
def test_fused_planes(pix, n_planes):
    """A fused frame of n planes with EWA in geometry B of the kernel matrix (source rect, output rect, fov 1.3): the three coordinate
    maps once, then one sampling pass per plane (3 + n launches: sony + digital_stretch has no filtered pre-pass and so no tail
    launch), each plane with its own background and plane_index equal to its own oracle render."""
    from tests.test_parity_gpu import _run_planes
    case = dict(w=75, h=43, ow=61, oh=37, fov=1.3, in_size=(83, 49), in_rect=(5, 4, 70, 40), out_size=(66, 41), out_rect=(4, 3, 62, 38),
                pix=pix, interp="EWA: Robidoux", lens="sony", digital="digital_stretch")
    bgv = lambda p, i: p.background.__setitem__(slice(0, 4), [0.1 * (i + 1), 0.5, 0.25, 1.0])
    outs, launches, _ = _run_planes(case, n_planes, vary=bgv)
    assert launches == 3 + n_planes, launches
    for i, (want, got) in enumerate(outs):
        assert np.array_equal(got, want), (pix, i, int((got != want).sum()))
