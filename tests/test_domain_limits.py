"""The packed warp kernel's domain windows on both sides of every boundary, and the warp at the limits of its frame geometry.

The packed kernel is exact only on frames that fit the windows its shortcuts were proven for (warp_kernel_x2.cuh): fill_uniforms and
plan_frame (csrc/c_abi.cu) and make_map (csrc/warp_kernel.cuh) send every other frame to the lean kernel (F_WILD) or drop one shortcut
(F_INTPRO, F_FILTER).  Each window is one comparison; a window that is off by one, or wider than its proof, renders wrong bytes only at
the shapes nobody renders.  BOUNDARIES has one row per window: the comparison it tests, a frame just inside and one just outside
(np.nextafter for float thresholds, +-1 for integer ones), and, written down here rather than read from the library, the feature bits
and the plan code each side must give.

CPU tests: every row through gf_cuda_plan_features (host-only: huge geometries need no allocation), and the rows that show the two
windows no frame can reach without another rule making it wild first.  GPU tests: both sides of every row rendered in every variant the
planner can give them (packed trusted and guarded, lean, general, Lanczos4, EWA where the footprint guard allows) byte for byte against
oracle_lib.undistort_image, guard bytes and launch counts checked; the source-rect rows proven to sample the last source pixel and past
it, the 131072-row frame proven to defer pairs in rows >= 65536; then frames whose byte offsets pass 2^31 and 2^32 (input, output,
two-pass coordinate map, checksums) and the 524280-row launch limit.
"""
import ctypes as C
import gc
import time

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi, synth
from tests import cases, oracle_lib
from tests.test_kernel_matrix import GUARD, MODES, _first_bad, report, set_switch

F = abi.F
W, H = 75, 43                     # the kernel matrix's odd size
FAKE_PTR = 1 << 40                # an aligned non-null address: gf_cuda_plan_features never dereferences a buffer
LENS_PAIRS = [("opencv_fisheye", None), ("poly3", None), ("sony", "digital_stretch"), ("gopro", "gopro_warp")]
LENS_PIX = ["RGBA8", "Luma16", "RGBAf"]
GEOM_PAIR = ("opencv_fisheye", None)
EWA_MODE = ("general-ewa", "GF_DISABLE_LEAN", "EWA: Mitchell", "host", 0x10)
VARIANTS = [m for m in MODES if m[0] in ("packed", "packed-guarded", "lean", "general", "packed-coords")]
K_BAND = [-0.42, 0.0, 0.0, 0.0] + [0.0] * 8          # tests/test_filter_queue.py: a cap inside a 4K frame, a band of corners defers
F32 = np.float32


def up(x):
    return float(np.nextafter(F32(x), F32(np.inf)))


def down(x):
    return float(np.nextafter(F32(x), F32(0.0)))


def bits(*names):
    out = 0
    for n in names:
        out |= F[n]
    return out


# ---- frames ---------------------------------------------------------------------------------------------------------------------
class Frame:
    """One warp call: KernelParams, pixel type, lens pair, input and output buffer geometry (width, height, stride, length) and, for
    rendering, the matrices.  Built from cases.build's frame (75 x 43, fov 1.3, rolling shutter) and then changed by `patch`."""

    def __init__(self, pix, lens, digital, patch=None, **case):
        base = dict(w=W, h=H, fov=1.3, pix=pix, lens=lens, digital=digital)
        base.update(case)
        p, _, m, _, _, _, _, _ = cases.build(base)
        self.p, self.m, self.pix, self.lens, self.digital = p, m, pix, lens, digital
        self.bpp = p.bytes_per_pixel
        bw, bh = base.get("in_size", (base["w"], base["h"]))
        obw, obh = base.get("out_size", (base.get("ow", base["w"]), base.get("oh", base["h"])))
        self.inb = [bw, bh, p.stride, bh * p.stride]
        self.outb = [obw, obh, p.output_stride, obh * p.output_stride]
        if patch:
            patch(self)

    def set_in(self, w, h, stride=None, rect=None):
        stride = stride or w * self.bpp
        self.p.stride = stride
        self.inb = [w, h, stride, h * stride]
        self.p.source_rect[:] = list(rect or (0, 0, w, h))
        self.p.flags |= abi.FLAG_HAS_SOURCE_RECT

    def set_out(self, ow, oh, w, h, stride=None, rect=None, rows=None):
        """Output frame ow x oh drawn into rect (default: the whole buffer) of a w x h buffer; rows: the buffer's length in rows."""
        stride = stride or w * self.bpp
        p = self.p
        fov = p.fov / (p.width / p.output_width)
        p.output_width, p.output_height, p.output_stride = ow, oh, stride
        p.fov = fov * (p.width / ow)
        p.output_rect[:] = list(rect or (0, 0, w, h))
        p.flags |= abi.FLAG_HAS_OUTPUT_RECT
        self.outb = [w, h, stride, (rows or h) * stride]

    def desc(self, which, ptr):
        w, h, stride, n = self.inb if which == "in" else self.outb
        d = abi.BufferDesc()
        d.width, d.height, d.stride, d.kind, d.ptr, d.len = w, h, stride, abi.BUF_DEVICE, ptr, n
        return d

    def plan(self, table_flags=0, src=FAKE_PTR, dst=FAKE_PTR):
        """(gf_cuda_plan_features code, feature word, gf_cuda_plan code)."""
        lib = g.load_library()
        i, o = self.desc("in", src), self.desc("out", dst)
        feat = C.c_uint32(0)
        args = (C.byref(self.p), abi.PIXEL_TYPES[self.pix][0], abi.LENS[self.lens], abi.LENS[self.digital] if self.digital else 0,
                C.byref(i), C.byref(o), 0, table_flags, 1)
        return lib.gf_cuda_plan_features(*args, C.byref(feat)), feat.value, lib.gf_cuda_plan(*args)


def setp(**kv):
    """A patch that sets KernelParams fields (arrays: {index: value})."""
    def patch(fr):
        for k, v in kv.items():
            if isinstance(v, dict):
                arr = getattr(fr.p, k)
                for i, x in v.items():
                    arr[i] = x
            else:
                setattr(fr.p, k, v)
    return patch


def chain(*patches):
    def patch(fr):
        for q in patches:
            q(fr)
    return patch


# ---- the boundary table ---------------------------------------------------------------------------------------------------------
# What a side must give: the plan code with tame host tables, bits that must be set and bits that must be clear.
PACKED = dict(code=3, has=0, lacks=bits("F_WILD"))
INTPRO = dict(code=3, has=bits("F_INTPRO"), lacks=bits("F_WILD"))
NO_INTPRO = dict(code=3, has=0, lacks=bits("F_WILD", "F_INTPRO"))
WILD = dict(code=1, has=bits("F_WILD"), lacks=bits("F_FILTER"))
FILTER = dict(code=3, has=bits("F_FILTER"), lacks=bits("F_WILD"))
NO_FILTER = dict(code=3, has=0, lacks=bits("F_WILD", "F_FILTER"))
REFUSED = dict(code=-1)                                # GF_ERR_BAD_PARAMS


class Boundary:
    """One window: `rule` cites the comparison; inside / outside are lists of (label, Frame factory, expectation); `render`: the GPU
    renders both sides (lens rows on LENS_PAIRS x LENS_PIX, geometry rows on their own frame); `ewa`: EWA is comparable."""

    def __init__(self, name, rule, inside, outside, render=True, ewa=True, lens_rows=False):
        self.name, self.rule, self.inside, self.outside = name, rule, inside, outside
        self.render, self.ewa, self.lens_rows = render, ewa, lens_rows

    def __repr__(self):
        return self.name


def lens_row(name, rule, field, index, inside, outside, extra_outside=(), pairs=None, ewa=True, extra_inside=()):
    """A KernelParams coefficient on LENS_PAIRS (or `pairs`): inside and outside values of p.<field>[index]."""
    def mk(v):
        return lambda pix, lens, digital, interp="Bilinear": Frame(pix, lens, digital, setp(**{field: {index: v}}), interp=interp)
    b = Boundary(name, rule, [("%r" % v, mk(v), PACKED) for v in (inside,) + tuple(extra_inside)], [("%r" % outside, mk(outside), WILD)] +
                 [("%r" % v, mk(v), WILD) for v in extra_outside], ewa=ewa, lens_rows=True)
    b.pairs = pairs or LENS_PAIRS
    return b


def geom(patch, pix="RGBA8", **case):
    return lambda interp="Bilinear": Frame(pix, GEOM_PAIR[0], GEOM_PAIR[1], patch, interp=interp, **case)


def wide_src(end):
    """A wide, 43-row input whose source rect ends at column `end` (the frame's 75 columns map onto the rect's 75)."""
    return lambda fr: fr.set_in(end, H, rect=(end - W, 0, W, H))


def tall_src(end):
    """A 75-pixel wide input of `end` rows whose source rect ends at row `end`."""
    return lambda fr: fr.set_in(W, end, rect=(0, end - H, W, H))


def frame_height(h):
    """A frame of h rows (the source-rect map's divisor) drawn from a 43-row source rect; the 43-row table is clamped as always."""
    return setp(height=h)


def out_origin(x0, scaled):
    """A 7 x 4 output frame drawn at column x0 of a 4-row output buffer 2^20 + 8 pixels wide: into a 7-pixel rect (identity map) or an
    8-pixel one (scaled).  Identity: (2^21 + 8) * 7 < 2^24, the identity test holds for every x0 here."""
    return lambda fr: fr.set_out(7, 4, (1 << 20) + 8, 4, rect=(x0, 0, 8 if scaled else 7, 4))


def out_origin_y(y0, scaled):
    return lambda fr: fr.set_out(8, 4, 8, 4, rect=(0, y0, 8, 5 if scaled else 4))


def out_origin_visible(x0):
    """A scaled output map with a negative origin x0 whose rect ends at column 8 of the 2^20 + 8 pixel wide buffer: columns 0..7 map
    into the 7-pixel output frame's last column, so they are written."""
    return lambda fr: fr.set_out(7, 4, (1 << 20) + 8, 4, rect=(x0, 0, 8 - x0, 4))


def out_origin_y_visible(y0):
    """The same on the y map: a rect from row y0 < 0 to row 4 of a 4-row buffer; every row maps into the 4-row output's last row."""
    return lambda fr: fr.set_out(8, 4, 8, 4, rect=(0, y0, 8, 4 - y0))


def out_width(ow, stride_px=None):
    return lambda fr: fr.set_out(ow, 4, ow, 4, stride=(stride_px or ow) * fr.bpp)


def out_height(oh):
    return lambda fr: fr.set_out(4, oh, 4, oh)


def filter_cols(stride):
    """Luma8, a 16384 x 4 output in a buffer of `stride` bytes per row (out_cols = stride)."""
    return lambda fr: fr.set_out(16384, 4, 16384, 4, stride=stride)


def filter_rows(rows, buffer_rows=None):
    """Luma8, a 3840 x 2160 output frame drawn into a 32-pixel wide rect of `rows` rows (a positive scale, so the packed kernel keeps
    it), the whole buffer (buffer_rows: the buffer ends there instead).  Every row is written, the last one included, so a pair at
    row 131072 that the queue could not address renders other bytes.  The source is a 3840 x 2160 frame with K_BAND, whose
    corner band defers pairs in the top and the bottom rows of the buffer alike."""
    def patch(fr):
        fr.set_out(3840, 2160, 32, rows, stride=32, rect=(0, 0, 32, rows), rows=buffer_rows)
    return patch


def launch_rows(rows):
    return lambda fr: fr.set_out(8, rows, 8, rows, stride=8)


BOUNDARIES = [
    lens_row("k[%d]" % i, "fill_uniforms: isfinite(k[i]) && |k[i]| <= 2^40", "k", i, 2.0 ** 40, up(2.0 ** 40),
             extra_outside=(float("inf"), float("nan")), ewa=False) for i in range(12)
] + [
    lens_row("translation2d[%d]%s" % (i, s), "fill_uniforms: |translation2d[i]| < 2^19", "translation2d", i, sg * down(2.0 ** 19), sg * 2.0 ** 19)
    for i in range(2) for s, sg in (("", 1.0), ("-", -1.0))
] + [
    # f == 0 is tame too: the packed kernel's trusted path then meets the infinite and NaN coordinates of a zero focal length
    lens_row("f[%d]-low" % i, "fill_uniforms: tame(f[i]), 2^-40 <= |f| (or f == 0)", "f", i, 2.0 ** -40, down(2.0 ** -40), ewa=False,
             extra_inside=(0.0,)) for i in range(2)
] + [
    lens_row("f[%d]-high" % i, "fill_uniforms: tame(f[i]), |f| <= 2^40", "f", i, 2.0 ** 40, up(2.0 ** 40), ewa=False) for i in range(2)
] + [
    lens_row("c[%d]%s" % (i, s), "fill_uniforms: |c[i]| >= 2^-10 (map_apply_x2's numerator window)", "c", i, sg * 2.0 ** -10, sg * down(2.0 ** -10))
    for i in range(2) for s, sg in (("", 1.0), ("-", -1.0))
] + [
    lens_row("gopro-k1-low", "fill_uniforms: gopro k1 tame and non-zero", "k", 1, 2.0 ** -40, down(2.0 ** -40), pairs=[("gopro", None), ("gopro", "gopro_warp")], ewa=False),
    lens_row("gopro-k1-high", "fill_uniforms: gopro k1 tame", "k", 1, 2.0 ** 40, up(2.0 ** 40), pairs=[("gopro", None), ("gopro", "gopro_warp")], ewa=False),
] + [
    lens_row("gopro_warp[%d]" % i, "fill_uniforms: gopro_warp digital_lens_params[i] finite and <= 2^40", "digital_lens_params", i, 2.0 ** 40,
             up(2.0 ** 40), pairs=[("gopro", "gopro_warp")], ewa=False) for i in range(16)
] + [
    Boundary("source-rect-end-x", "fill_uniforms: src_rect[2] <= 2^16 (8-bit sampler: rounding word and interior test)",
             [("65536", geom(wide_src(65536), fov=2.0), PACKED)], [("65537", geom(wide_src(65537), fov=2.0), WILD)]),
    Boundary("source-rect-end-y", "fill_uniforms: src_rect[3] <= 2^16",
             [("65536", geom(tall_src(65536), fov=2.0), PACKED)], [("65537", geom(tall_src(65537), fov=2.0), WILD)]),
    Boundary("source-map-divisor", "fill_uniforms smap_ok: frame_h (smap_y.div) <= 2^20",
             [("2^20", geom(frame_height(1 << 20)), PACKED)], [("2^20+1", geom(frame_height((1 << 20) + 1)), WILD)]),
    Boundary("output-origin-x-identity", "fill_uniforms: F_INTPRO iff |omap.in_min| < 2^20; int_map_ok: an identity map passes at any in_min",
             [("2^20-1", geom(out_origin((1 << 20) - 1, False)), INTPRO)],
             [("2^20", geom(out_origin(1 << 20, False)), NO_INTPRO), ("2^20+1", geom(out_origin((1 << 20) + 1, False)), NO_INTPRO),
              ("-(2^20-1)", geom(out_origin(-(1 << 20) + 1, False)), INTPRO), ("-2^20", geom(out_origin(-(1 << 20), False)), NO_INTPRO)]),
    Boundary("output-origin-x-scaled", "fill_uniforms int_map_ok: a scaled map needs |in_min| <= 2^20",
             [("2^20-1", geom(out_origin((1 << 20) - 1, True)), NO_INTPRO), ("2^20", geom(out_origin(1 << 20, True)), NO_INTPRO),
              ("-2^20", geom(out_origin(-(1 << 20), True)), NO_INTPRO), ("-2^20 written", geom(out_origin_visible(-(1 << 20))), NO_INTPRO)],
             [("2^20+1", geom(out_origin((1 << 20) + 1, True)), WILD), ("-(2^20+1)", geom(out_origin(-(1 << 20) - 1, True)), WILD),
              ("-(2^20+1) written", geom(out_origin_visible(-(1 << 20) - 1)), WILD)]),
    Boundary("output-origin-y", "fill_uniforms: the same windows on the y map (a positive origin is past the buffer: nothing is written)",
             [("2^20-1", geom(out_origin_y((1 << 20) - 1, False)), INTPRO), ("2^20 scaled", geom(out_origin_y(1 << 20, True)), NO_INTPRO),
              ("-2^20 scaled, written", geom(out_origin_y_visible(-(1 << 20))), NO_INTPRO)],
             [("2^20", geom(out_origin_y(1 << 20, False)), NO_INTPRO), ("2^20+1 scaled", geom(out_origin_y((1 << 20) + 1, True)), WILD),
              ("-(2^20+1) scaled", geom(out_origin_y(-(1 << 20) - 1, True)), WILD),
              ("-(2^20+1) scaled, written", geom(out_origin_y_visible(-(1 << 20) - 1)), WILD)]),
    Boundary("identity-width", "make_map: (out_cols + |x0|) * output_width < 2^24",
             [("4095", geom(out_width(4095)), INTPRO)], [("4096", geom(out_width(4096)), NO_INTPRO)]),
    Boundary("identity-height", "make_map: (out_rows + |y0|) * output_height < 2^24",
             [("4095", geom(out_height(4095)), INTPRO)], [("4096", geom(out_height(4096)), NO_INTPRO)]),
    Boundary("identity-stride-padding", "make_map: out_cols = output_stride / bpp counts the padding",
             [("4000 in 4194", geom(out_width(4000, 4194)), INTPRO)], [("4000 in 4195", geom(out_width(4000, 4195)), NO_INTPRO)]),
    Boundary("filter-cols", "plan_frame: out_cols <= X2Filter::kMaxCols (2^16)",
             [("65536", geom(filter_cols(65536), pix="Luma8"), FILTER)], [("65537", geom(filter_cols(65537), pix="Luma8"), NO_FILTER)]),
    Boundary("filter-rows", "plan_frame: out_rows <= X2Filter::kMaxRows (2^17)",
             [("131072", geom(filter_rows(131072), pix="Luma8", w=3840, h=2160, params=dict(k=K_BAND)), FILTER)],
             [("131073", geom(filter_rows(131073), pix="Luma8", w=3840, h=2160, params=dict(k=K_BAND)), NO_FILTER)]),
    Boundary("launch-rows", "validate: ceil(len / output_stride) <= 65535 * GF_BLOCK_Y = 524280",
             [("524280", geom(launch_rows(524280), pix="Luma8"), NO_INTPRO)], [("524281", geom(launch_rows(524281), pix="Luma8"), REFUSED)],
             render=False),
]
BY_NAME = {b.name: b for b in BOUNDARIES}


def sides(b):
    """(row, side, label, factory, expectation, pair) of a boundary: lens rows once per pair."""
    for side, lst in (("inside", b.inside), ("outside", b.outside)):
        for label, mk, exp in lst:
            if b.lens_rows:
                for lens, digital in b.pairs:
                    yield side, label, (lambda pix, interp="Bilinear", mk=mk, lens=lens, digital=digital: mk(pix, lens, digital, interp)), exp, (lens, digital)
            else:
                yield side, label, (lambda pix, interp="Bilinear", mk=mk: mk(interp)), exp, GEOM_PAIR


def check_side(fr, exp, where):
    code, feat, code2 = fr.plan()
    assert code == code2, (where, code, code2)
    assert code == exp["code"], (where, "plan code", code, exp["code"])
    if code < 0:
        return
    assert feat & exp["has"] == exp["has"], (where, "missing bits", hex(exp["has"] & ~feat))
    assert feat & exp["lacks"] == 0, (where, "unexpected bits", hex(feat & exp["lacks"]))


# ---- the table, without a GPU ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [b.name for b in BOUNDARIES])
def test_boundary(monkeypatch, name):
    """Both sides of the window through gf_cuda_plan_features and gf_cuda_plan: the declared plan code and bits (RGBA8; lens rows on
    every pair they apply to)."""
    set_switch(monkeypatch, None)
    b = BY_NAME[name]
    n = {"inside": 0, "outside": 0}
    for side, label, mk, exp, pair in sides(b):
        pix = "RGBA8"
        fr = mk(pix)
        check_side(fr, exp, (b.name, b.rule, side, label, pair))
        n[side] += 1
    assert n["inside"] and n["outside"]


def test_every_window_has_a_row():
    """The windows the packed kernel's proofs need, each with a row (the masked ones below have theirs)."""
    rules = " ".join(b.rule for b in BOUNDARIES)
    for needle in ("|k[i]| <= 2^40", "translation2d", "tame(f[i])", "|c[i]| >= 2^-10", "gopro k1", "gopro_warp", "src_rect[2] <= 2^16",
                   "src_rect[3] <= 2^16", "<= 2^20", "< 2^20", "< 2^24", "kMaxCols", "kMaxRows", "524280"):
        assert needle in rules, needle


def test_interior_span_window_is_masked(monkeypatch):
    """fill_uniforms' interior_span >= 2^17 cannot decide a frame: a span of 2^17 needs a source rect ending at 2^17 + 2 or later (span = end - 2 - origin, origin >= 0), which the
    source-rect end rule (src_rect[2], src_rect[3] <= 2^16) makes wild first.  The widest rect the end rule lets through has a span of
    2^16 - 2 and stays packed."""
    set_switch(monkeypatch, None)
    for end, exp in (((1 << 16), PACKED), ((1 << 17) + 2, WILD)):
        check_side(Frame("RGBA8", *GEOM_PAIR, lambda fr, end=end: fr.set_in(end, H, rect=(0, 0, end, H))), exp, ("span x", end))
        check_side(Frame("RGBA8", *GEOM_PAIR, lambda fr, end=end: fr.set_in(W, end, rect=(0, 0, W, end))), exp, ("span y", end))
    # the end rule alone: a rect ending at 2^16 + 1 (span 2^16 - 1, far below 2^17) is already wild
    check_side(Frame("RGBA8", *GEOM_PAIR, lambda fr: fr.set_in((1 << 16) + 1, H, rect=(0, 0, (1 << 16) + 1, H))), WILD, "end rule")


def test_rs_lim_window_is_masked(monkeypatch):
    """fill_uniforms' rs_lim >= 2^22 cannot decide a frame: rs_lim is the frame's height (vertical readout), and any height above 2^20
    is wild by the source-map divisor rule (smap_y.div <= 2^20); with horizontal readout it is the width, which validate caps at 16384."""
    set_switch(monkeypatch, None)
    for h in ((1 << 20) + 1, (1 << 22) - 1, 1 << 22):
        check_side(Frame("RGBA8", *GEOM_PAIR, frame_height(h)), WILD, ("height", h))
    fr = Frame("RGBA8", *GEOM_PAIR, chain(setp(width=16385), lambda fr: setattr(fr.p, "flags", fr.p.flags | abi.FLAG_HORIZONTAL_RS)))
    check_side(fr, REFUSED, "horizontal readout, width 16385")


def test_plan_refuses_what_the_call_refuses(monkeypatch):
    """gf_cuda_plan / gf_cuda_plan_features and gf_cuda_create share validate: an output of 524281 rows is GF_ERR_BAD_PARAMS for all of
    them (the launch has at most 65535 row blocks of 8 rows); so is an output stride shorter than one pixel."""
    set_switch(monkeypatch, None)
    lib = g.load_library()
    fr = Frame("Luma8", *GEOM_PAIR, launch_rows(524281))
    assert fr.plan()[0] == -1 and fr.plan()[2] == -1
    h = C.c_void_p()
    i, o = fr.desc("in", FAKE_PTR), fr.desc("out", FAKE_PTR)
    assert lib.gf_cuda_create(C.byref(h), 0, C.byref(fr.p), abi.PIXEL_TYPES["Luma8"][0], abi.LENS[GEOM_PAIR[0]], 0, C.byref(i), C.byref(o), 0) == -1
    assert not h.value
    fr = Frame("RGBA8", *GEOM_PAIR, lambda fr: fr.set_out(4, 4, 1, 8, stride=3))
    assert fr.plan()[0] == -1


# ---- rendering ------------------------------------------------------------------------------------------------------------------
def _aligned(n, fill):
    raw = np.full(n + 64, fill, np.uint8) if fill else np.zeros(n + 64, np.uint8)
    off = (-raw.ctypes.data) % 64
    return raw[off:off + n]


def source(fr):
    """The input buffer: zeros, with synthetic content in the source rect's rows and columns only (the rest is never read, and zero
    pages cost nothing)."""
    w, h, stride, n = fr.inb
    src = _aligned(n, 0)
    x0, y0, rw, rh = list(fr.p.source_rect)
    img = synth.synthetic_frame(rw, rh, fr.pix, stride=rw * fr.bpp).reshape(rh, rw * fr.bpp)
    rows = src.reshape(h, stride) if n == h * stride else None
    rows[y0:y0 + rh, x0 * fr.bpp:(x0 + rw) * fr.bpp] = img
    return src


def oracle(fr, src):
    want = _aligned(fr.outb[3], 0xA5)
    assert oracle_lib.undistort_image(src, want, fr.p, fr.pix, fr.lens, fr.digital, fr.m) == 0
    return want


def expected_code(exp, mode):
    """The plan code a side gives under one variant: WILD sides take the lean kernel where the packed one would run."""
    _, switch, interp, tables, code = mode
    if exp is WILD and (code & 0xF) >= 1:
        return (code & 0x10) | (0 if switch == "GF_DISABLE_LEAN" else 1)
    return code


def launches_of(fr, code, interp, tables, src_ptr, dst_ptr):
    n = 1 if interp == "Bilinear" else (4 if interp.startswith("EWA") else 2)
    if (code & 0xF) >= 2:          # device tables without a verdict still run the filtered pre-pass; as trusted as tame host tables
        _, feat, _ = fr.plan(0, src_ptr, dst_ptr)
        n += 1 if feat & F["F_FILTER"] else 0
    return n


def render_dev(fr, tsrc, mode, sentinel=0xA5, tdst=None):
    """Render fr (DEVICE buffers) under one variant; returns (output incl. GUARD bytes as numpy, launches, plan code)."""
    import torch
    _, _, interp, tables, _ = mode
    n = fr.outb[3]
    if tdst is None:
        tdst = torch.full((n + GUARD,), sentinel, dtype=torch.uint8, device="cuda")
    host_flags = g.load_library().gf_table_flags_host(fr.m.ctypes.data, fr.m.shape[0])
    code = fr.plan(host_flags if tables == "host" else 1)[2]
    bufs = g.Buffers(g.BufferDescription(tuple(fr.inb[:3]), tsrc.data_ptr(), length=fr.inb[3]),
                     g.BufferDescription(tuple(fr.outb[:3]), tdst.data_ptr(), length=n))
    ctx = g.CudaWrapper.new(fr.p, fr.pix, fr.lens, fr.digital, bufs)
    try:
        torch.cuda.synchronize()
        l0 = ctx.launch_count
        if tables == "host":
            ctx.undistort_image(bufs, g.FrameTransform(matrices=fr.m, kernel_params=fr.p))
        else:
            tm = torch.from_numpy(fr.m).cuda()
            ctx.undistort_image_dev(bufs, fr.p, tm.data_ptr(), fr.m.shape[0])
        ctx.synchronize()
        launches = ctx.launch_count - l0
    finally:
        ctx.close()
    return tdst, launches, code


def compare(where, fr, tdst, want, bad):
    got = tdst.cpu().numpy()
    n = fr.outb[3]
    if not np.array_equal(got[n:], np.full(GUARD, 0xA5, np.uint8)):
        bad.append("%s: wrote past the end of the output" % (where,))
    elif not np.array_equal(got[:n], want):
        bad.append("%s: %d bytes differ, first at %s" % (where, int((got[:n] != want).sum()), _first_bad(want, got[:n], fr.p.output_stride, fr.bpp)))


def render_sides(request, monkeypatch, boundaries, pixel_types, label):
    """Render every side of `boundaries` in every variant; a wrong plan code or launch count is a failure like wrong bytes, but the bytes
    are still compared, so that the report says which renders differ from the oracle.  Reports each failing render (up to 64)."""
    import torch
    t0 = time.perf_counter()
    renders, bad, plan_bad, per_row = 0, [], [], {}
    for b in boundaries:
        modes = VARIANTS + ([EWA_MODE] if b.ewa else [])
        for side, lbl, mk, exp, (lens, digital) in sides(b):
            for pix in (pixel_types if b.lens_rows else [None]):
                wants = {}                                      # the oracle once per (row, side, pair, pixel type, resampler)
                for mode in modes:
                    set_switch(monkeypatch, mode[1])
                    fr = mk(pix, mode[2])
                    if mode[2] not in wants:
                        src = source(fr)
                        wants[mode[2]] = (src, oracle(fr, src))
                    src, want = wants[mode[2]]
                    tsrc = torch.from_numpy(src).cuda()
                    tdst, launches, code = render_dev(fr, tsrc, mode)
                    where = (b.name, side, lbl, lens, digital, fr.pix, mode[0])
                    want_l = launches_of(fr, code, mode[2], mode[3], tsrc.data_ptr(), tdst.data_ptr())
                    if code != expected_code(exp, mode) or launches != want_l:
                        plan_bad.append("%s: plan code %d (want %d), %d launches (want %d)" % (where, code, expected_code(exp, mode), launches, want_l))
                    compare(where, fr, tdst, want, bad)
                    renders += 1
                    per_row[b.name] = per_row.get(b.name, 0) + 1
                    del tsrc, tdst
    report(request, "%s: %d renders, %d with other bytes than the oracle's, %d with another plan or launch count, %.1f s; renders per row: %s" %
           (label, renders, len(bad), len(plan_bad), time.perf_counter() - t0, ", ".join("%s %d" % kv for kv in per_row.items())))
    for line in (bad + plan_bad)[:64]:
        report(request, "  " + line)
    assert not bad and not plan_bad, "%d renders with other bytes, %d with another plan; first: %s" % (len(bad), len(plan_bad), (bad + plan_bad)[0])
    return renders


@pytest.mark.gpu
def test_lens_rows_render(request, monkeypatch):
    """Lens coefficient, translation, focal length and principal point rows: both sides on their pairs in RGBA8, Luma16 and RGBAf, in
    every variant, byte for byte against the oracle.  EWA on the rows whose values keep the Jacobian probes' footprints inside the
    kernel's 2^22-tap guard (the k, f and gopro rows at 2^40 give footprints the guard renders as background, as documented in
    warp_kernel.cuh)."""
    rows = [b for b in BOUNDARIES if b.lens_rows]
    assert render_sides(request, monkeypatch, rows, LENS_PIX, "test_lens_rows_render") > 2000


@pytest.mark.gpu
def test_geometry_rows_render(request, monkeypatch):
    """Source-rect end, source-map divisor, output-rect origin, identity cut-off and filter rows: both sides in every variant against
    the oracle."""
    rows = [b for b in BOUNDARIES if not b.lens_rows and b.render]
    assert render_sides(request, monkeypatch, rows, None, "test_geometry_rows_render") > 100


@pytest.mark.parametrize("axis", ["x", "y"])
def test_source_rect_rows_reach_their_edge(axis):
    """The inside frame of each source-rect row (fov 2: the frame's edge is in view) samples source coordinates in [65535, 65536) (the
    last pixel the 8-bit sampler's rounding word and interior test cover) and past 65536 (background), per oracle_lib.undistort_coord."""
    b = BY_NAME["source-rect-end-" + axis]
    fr = b.inside[0][1]()
    i = 0 if axis == "x" else 1
    at_edge = past = 0
    for y in range(fr.p.output_height):
        for x in range(fr.p.output_width):
            s = oracle_lib.undistort_coord(x, y, fr.p, fr.m, fr.lens, fr.digital)
            if s is None:
                continue
            at_edge += 65535.0 <= s[i] < 65536.0
            past += s[i] >= 65536.0
    assert at_edge > 0 and past > 0, (axis, at_edge, past)


@pytest.mark.gpu
def test_filter_rows_defer_past_row_65536(request, monkeypatch):
    """The 131072-row frame defers pairs in rows >= 65536, where bit 31 of a queue entry x | (y0 / 2) << 16 is set: its deferral count
    (gf_cuda_filter_stats, no more than the queue holds, so every pair went through the queue and its tail launch) exceeds that of the
    same frame in an output buffer that ends at row 65536, and both render the oracle's bytes."""
    import torch
    set_switch(monkeypatch, None)
    counts = {}
    for name, buffer_rows in (("full", None), ("first 65536 rows", 65536)):
        fr = Frame("Luma8", *GEOM_PAIR, lambda f: filter_rows(131072, buffer_rows)(f), w=3840, h=2160, params=dict(k=K_BAND))
        code, feat, _ = fr.plan()
        assert code == 3 and feat & F["F_FILTER"], (name, code, hex(feat))
        src = source(fr)
        want = oracle(fr, src)
        tsrc = torch.from_numpy(src).cuda()
        tdst = torch.full((fr.outb[3] + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
        bufs = g.Buffers(g.BufferDescription(tuple(fr.inb[:3]), tsrc.data_ptr(), length=fr.inb[3]),
                         g.BufferDescription(tuple(fr.outb[:3]), tdst.data_ptr(), length=fr.outb[3]))
        ctx = g.CudaWrapper.new(fr.p, fr.pix, fr.lens, fr.digital, bufs)
        try:
            ctx.undistort_image(bufs, g.FrameTransform(matrices=fr.m, kernel_params=fr.p))
            s = ctx.filter_stats()
        finally:
            ctx.close()
        bad = []
        compare(name, fr, tdst, want, bad)
        assert not bad, bad
        assert s["frames"] == 1 and s["count"] <= s["cap"], s        # every deferred pair went through the queue
        counts[name] = s["count"]
    report(request, "test_filter_rows_defer_past_row_65536: deferred pairs %s" % counts)
    assert counts["full"] > counts["first 65536 rows"] > 0, counts


# ---- frames past 2^31 and 2^32 bytes --------------------------------------------------------------------------------------------
GIB = 1 << 30


def need(request, dev_bytes, host_bytes=0):
    """Skip (with the reason printed) unless the device has dev_bytes free plus 1 GiB; the limits of this file are 12 GiB of device
    and 16 GiB of host memory at a time."""
    import torch
    assert dev_bytes <= 12 * GIB and host_bytes <= 16 * GIB
    gc.collect(); torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < dev_bytes + GIB:
        msg = "%s: %.1f GiB of device memory free, %.1f GiB needed" % (request.node.name, free / GIB, (dev_bytes + GIB) / GIB)
        report(request, "SKIP " + msg)
        pytest.skip(msg)
    return free


def big_input(interp="Bilinear"):
    """RGBA8, stride 65600 and 65536 rows (4.3 GB); the 75 x 43 frame's source rect ends at row 65536, so that its origin's byte
    offset (the packed gather's hot.src) passes 2^32."""
    return Frame("RGBA8", *GEOM_PAIR, lambda fr: fr.set_in(16400, 65536, stride=65600, rect=(16000, 65536 - H, W, H)), interp=interp)


@pytest.mark.gpu
def test_input_past_4gib(request, monkeypatch):
    """The 4.3 GB input in every variant (packed trusted and guarded, lean, general, Lanczos4) from a DEVICE buffer, then once through
    gf_cuda_undistort_image from a HOST buffer page-locked by gf_cuda_host_register: the oracle's bytes every time."""
    import torch
    fr = big_input()
    n = fr.inb[3]
    assert (65536 - H) * 65600 > 1 << 32 and n > 1 << 32
    need(request, n + (1 << 20), host_bytes=n)      # both parts: one 4.3 GB device buffer at a time; the HOST part pins n host bytes
    t0 = time.perf_counter()
    src = source(fr)                                           # only the rect's 43 rows are touched
    tsrc = torch.zeros(n, dtype=torch.uint8, device="cuda")
    lo = (65536 - H) * 65600
    tsrc[lo:].copy_(torch.from_numpy(src[lo:]))
    bad, renders = [], 0
    wants = {}
    for mode in VARIANTS:
        set_switch(monkeypatch, mode[1])
        f = big_input(mode[2])
        if mode[2] not in wants:
            wants[mode[2]] = oracle(f, src)
        tdst, launches, code = render_dev(f, tsrc, mode)
        assert code == mode[4], (mode, code)
        assert launches == launches_of(f, code, mode[2], mode[3], tsrc.data_ptr(), tdst.data_ptr()), (mode, launches)
        compare(("input past 4 GiB", mode[0]), f, tdst, wants[mode[2]], bad)
        renders += 1
    del tsrc, tdst
    gc.collect(); torch.cuda.empty_cache()
    assert not bad, bad                             # the DEVICE renders are settled before the HOST part may skip
    # one HOST call: the input page-locked in place, staged whole by the context
    set_switch(monkeypatch, None)
    need(request, n + (1 << 20), host_bytes=n)
    g.host_register(src)
    try:
        dst = _aligned(fr.outb[3], 0xA5)
        bufs = g.Buffers(g.BufferDescription(tuple(fr.inb[:3]), src), g.BufferDescription(tuple(fr.outb[:3]), dst))
        ctx = g.CudaWrapper.new(fr.p, fr.pix, fr.lens, fr.digital, bufs)
        try:
            ctx.undistort_image(bufs, g.FrameTransform(matrices=fr.m, kernel_params=fr.p))
        finally:
            ctx.close()
    finally:
        g.host_unregister(src)
    if not np.array_equal(dst, wants["Bilinear"]):
        bad.append("HOST call: %d bytes differ" % int((dst != wants["Bilinear"]).sum()))
    renders += 1
    del src
    report(request, "test_input_past_4gib: %d renders, %d failing, %.1f s, largest device allocation %.2f GiB" %
           (renders, len(bad), time.perf_counter() - t0, n / GIB))
    assert not bad, bad


def corner_output(interp="Bilinear"):
    """RGBAf: a 75 x 43 output frame in the bottom-right corner of a 16400 x 16416 output buffer (4.3 GB, stride 262400): the rect's
    bytes start past 2^32, and its two-pass coordinate map entries (8 bytes per buffer pixel, 2.15 GB) past 2^31."""
    return Frame("RGBAf", *GEOM_PAIR, lambda fr: fr.set_out(W, H, 16400, OUT_ROWS, rect=(16400 - W, OUT_ROWS - H, W, H)), interp=interp)


OUT_ROWS = 16416
CHUNK = 1 << 28


def count_not(a, lo, hi, value):
    """Bytes of a[lo:hi] (numpy or torch) that differ from `value`, in chunks of CHUNK bytes (the comparison's temporaries stay small)."""
    n = 0
    for i in range(lo, hi, CHUNK):
        d = a[i:min(hi, i + CHUNK)] != value
        n += int(d.sum().item() if hasattr(d, "item") else d.sum())
    return n


@pytest.mark.gpu
def test_output_past_4gib(request, monkeypatch):
    """Every variant (Lanczos4: its 2.15 GB coordinate map) renders the corner rect's bytes as the oracle does, and every byte outside
    the rect keeps its sentinel."""
    import torch
    fr = corner_output()
    n, stride = fr.outb[3], fr.outb[2]
    first = (OUT_ROWS - H) * stride + (16400 - W) * 16
    assert first > 1 << 32 and ((OUT_ROWS - H) * 16400 + 16400 - W) * 8 > 1 << 31
    # output, coordinate map and the chunked comparison's temporaries (CHUNK bytes and as many bools)
    need(request, n + GUARD + 16400 * OUT_ROWS * 8 + 2 * CHUNK + (1 << 20), host_bytes=n)
    t0 = time.perf_counter()
    src = source(fr)
    lo = (OUT_ROWS - H) * stride
    wants = {}                                                     # the oracle once per resampler, in the full buffer (4.3 GB of host memory)
    for interp in sorted({m[2] for m in VARIANTS}):
        f = corner_output(interp)
        want = _aligned(n, 0xA5)
        assert oracle_lib.undistort_image(src, want, f.p, f.pix, f.lens, f.digital, f.m) == 0
        assert count_not(want, 0, lo, 0xA5) == 0
        wants[interp] = want[lo:].copy()
        del want
    tsrc = torch.from_numpy(src).cuda()
    bad, renders = [], 0
    tdst = torch.empty(n + GUARD, dtype=torch.uint8, device="cuda")
    for mode in VARIANTS:
        set_switch(monkeypatch, mode[1])
        f = corner_output(mode[2])
        want_rows = wants[mode[2]]
        tdst.fill_(0xA5)
        tdst, launches, code = render_dev(f, tsrc, mode, tdst=tdst)
        assert code == mode[4], (mode, code)
        assert launches == launches_of(f, code, mode[2], mode[3], tsrc.data_ptr(), tdst.data_ptr()), (mode, launches)
        outside = count_not(tdst, 0, lo, 0xA5) + count_not(tdst, n, n + GUARD, 0xA5)
        got = tdst[lo:n].cpu().numpy()
        if outside:
            bad.append("%s: %d bytes outside the rect's rows written" % (mode[0], outside))
        elif not np.array_equal(got, want_rows):
            bad.append("%s: %d bytes differ" % (mode[0], int((got != want_rows).sum())))
        renders += 1
    del tsrc, tdst
    gc.collect(); torch.cuda.empty_cache()
    report(request, "test_output_past_4gib: %d renders, %d failing, %.1f s, largest device allocation %.2f GiB (+ %.2f GiB coordinate map)" %
           (renders, len(bad), time.perf_counter() - t0, n / GIB, 16400 * OUT_ROWS * 8 / GIB))
    assert not bad, bad


def checksum_chunks(parts, total):
    """sum(word[i] * (2 i + 1)) mod 2^64 of a byte string that is zero except for `parts` [(string offset, bytes)], summed up to
    4 * (total // 4) bytes: each part padded to whole words with the zeros around it."""
    s = 0
    end = total & ~3
    for off, b in parts:
        b = b[:max(0, end - off)]
        lead = off & 3
        w = np.concatenate([np.zeros(lead, np.uint8), b, np.zeros((-(lead + b.size)) % 4, np.uint8)]).view(np.uint32).astype(np.uint64)
        k = (np.arange(w.size, dtype=np.uint64) + np.uint64(off >> 2)) * np.uint64(2) + np.uint64(1)
        with np.errstate(over="ignore"):
            s = (s + int((w * k).sum(dtype=np.uint64))) % (1 << 64)
    return s


@pytest.mark.gpu
def test_checksums_past_4gib(request):
    """gf_cuda_checksum_dev over 2^33 + 4099 bytes (word indices past 2^31, byte offsets past 2^32 and 2^33) and
    gf_cuda_checksum_planes_dev with rows * stride > 2^32, against a chunked host restatement of checksum_host."""
    import torch
    lib = g.load_library()
    n = (1 << 33) + 4099
    need(request, n)
    t0 = time.perf_counter()
    rng = np.random.default_rng(7)
    buf = torch.zeros(n, dtype=torch.uint8, device="cuda")
    parts = []
    # disjoint parts, one inside the rows of the second plane descriptor below, the last one to the end
    for off in (0, (1 << 31) - 777, (1 << 32) - 4096 + 3, (1 << 32) + 12345 + 4096 * 500 - 300, (1 << 33) - 9001, n - 3000):
        b = rng.integers(0, 256, min(8192, n - off), dtype=np.uint8)
        buf[off:off + b.size].copy_(torch.from_numpy(b))
        parts.append((off, b))
    out = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.gf_cuda_checksum_dev(buf.data_ptr(), n, out.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert int(out.item()) % (1 << 64) == checksum_chunks(parts, n)
    # two descriptors: 65537 rows of 65598 bytes, 65600 apart (4.3 GB), then 1000 rows of 1001 bytes from 2^32 + 12345, whose rows
    # 499..501 hold random bytes
    descs = [(buf.data_ptr(), 65598, 65600, 65537), (buf.data_ptr() + (1 << 32) + 12345, 1001, 4096, 1000)]
    arr = (abi.ChecksumPlane * 2)(*[abi.ChecksumPlane(p, rb, st, r) for p, rb, st, r in descs])
    assert lib.gf_cuda_checksum_planes_dev(arr, 2, out.data_ptr(), None) == 0
    torch.cuda.synchronize()
    sparts, soff = [], 0
    for p, rb, st, r in descs:
        base = p - buf.data_ptr()
        for r0 in range(r):
            a = base + r0 * st
            if any(o < a + rb and a < o + b.size for o, b in parts):        # rows that hold non-zero bytes
                sparts.append((soff + r0 * rb, buf[a:a + rb].cpu().numpy()))
        soff += r * rb
    assert 65537 * 65600 > 1 << 32
    assert any(o >= 65537 * 65598 for o, _ in sparts)                  # the second descriptor sums non-zero rows
    assert int(out.item()) % (1 << 64) == checksum_chunks(sparts, soff)
    del buf
    gc.collect(); torch.cuda.empty_cache()
    report(request, "test_checksums_past_4gib: %.1f s, largest device allocation %.2f GiB" % (time.perf_counter() - t0, n / GIB))


@pytest.mark.gpu
def test_launch_row_limit(request, monkeypatch):
    """A 524280-row output renders the oracle's bytes; a 524281-row output (the same context) is GF_ERR_BAD_PARAMS before anything is
    enqueued: no launch, the output untouched."""
    import torch
    set_switch(monkeypatch, None)
    fr = BY_NAME["launch-rows"].inside[0][1]()
    src = source(fr)
    want = oracle(fr, src)
    tsrc = torch.from_numpy(src).cuda()
    bad = []
    for mode in VARIANTS:
        set_switch(monkeypatch, mode[1])
        f = BY_NAME["launch-rows"].inside[0][1](mode[2])
        w = want if mode[2] == "Bilinear" else oracle(f, src)
        tdst, launches, code = render_dev(f, tsrc, mode)
        assert code == mode[4] and launches == launches_of(f, code, mode[2], mode[3], tsrc.data_ptr(), tdst.data_ptr()), (mode, code, launches)
        compare(("524280 rows", mode[0]), f, tdst, w, bad)
    assert not bad, bad
    set_switch(monkeypatch, None)
    big = BY_NAME["launch-rows"].outside[0][1]()
    tdst = torch.full((big.outb[3] + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    bufs = g.Buffers(g.BufferDescription(tuple(fr.inb[:3]), tsrc.data_ptr(), length=fr.inb[3]),
                     g.BufferDescription(tuple(fr.outb[:3]), tdst.data_ptr(), length=fr.outb[3]))
    ctx = g.CudaWrapper.new(fr.p, fr.pix, fr.lens, fr.digital, bufs)
    try:
        torch.cuda.synchronize()
        l0 = ctx.launch_count
        bufs.output.length = big.outb[3]
        with pytest.raises(g.GyroflowCoreError) as e:
            ctx.undistort_image(bufs, g.FrameTransform(matrices=fr.m, kernel_params=fr.p))
        assert e.value.code == -1
        ctx.synchronize()
        assert ctx.launch_count == l0
    finally:
        ctx.close()
    assert int((tdst != 0xA5).sum().item()) == 0
