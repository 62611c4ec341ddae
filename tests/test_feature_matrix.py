"""Every bit of the warp's per-frame feature word, on every lens pair and kernel variant, against the CPU oracle.

fill_uniforms (csrc/c_abi.cu) turns a frame's KernelParams and buffers into a feature word (the F_* bits of csrc/warp_kernel.cuh,
mirrored as abi.F).  The word picks the kernel that renders the frame (plan_frame: general, lean, packed trusted / guarded, two-pass)
and the run-time branches of the general kernel.  test_kernel_matrix renders every (pair, pixel type, variant) with one set of
parameters; this file renders ROWS: each row is a cases.build override of one base frame (the kernel matrix's odd 75 x 43, fov 1.3 so
that no fov factor cancels, rolling shutter on), and states, independently of the library, the bits it adds to or removes from the
base frame's word and its class, i.e. which kernel must render it:

  general   a general-only feature (F_GENERAL_ONLY), a digital lens with flag bit 2 clear, or unaligned pixel access: the general kernel
  guarded   IBIS rows in the matrix table: the packed kernel on its guarded path
  lean      F_WILD: the lean kernel
  packed    anything else: the packed kernel, on its trusted path with tame host tables

CPU tests: through gf_cuda_plan_features every row sets exactly the bits it declares, and the rows together change every bit of the
enum; gf_cuda_plan returns the code the row's class predicts under every switch of MODES; every row changes the oracle's output except
the declared no-ops, which keep it byte for byte; the rows no other test restates agree with tests/np_restatement.py.  GPU tests:
every cell byte for byte against oracle_lib.undistort_image, with guard bytes after the output and the launch count checked.
"""
import ctypes as C
import os
import re
import time
import warnings

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi
from tests import cases, oracle_lib
from tests.test_kernel_matrix import (GUARD, H, MODES, PIXEL_TYPES, W, _bpp_align, _first_bad, build, descs, geometries, library_pairs,
                                      render, report, set_switch)

MODES = [m for m in MODES if not m[2].startswith("EWA")]       # the seven bilinear / Lanczos4 variants; EWA rows run EWA_MODE only
F = abi.F
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEN_PIX = ["RGBA8", "Luma16", "RGBAf"]                          # one 8-bit, one 16-bit, one float layout
PIXEL_PAIRS = [("opencv_fisheye", None), ("sony", "digital_stretch"), ("gopro", "gopro_warp")]
GEN_MODES = [MODES[3], MODES[6]]                                # general (fused bilinear) and general-coords (Lanczos4)
EWA_MODE = ("general-ewa", None, "EWA: Mitchell", "host", 0x10)
NOOP_LENSES = ("opencv_fisheye", "sony", "generic_polynomial", "gopro")     # the models with an "all coefficients zero" early-out
BG = [0.25, 0.5, 0.75, 1.0]


def bits(*names):
    out = 0
    for n in names:
        out |= F[n]
    return out


class Row:
    """One row of the table.  case: cases.build keys, or a function of (lens, digital, pix) returning them; add / remove: F_* bits
    relative to the base frame's word (ints or functions of (lens, digital, pix)); cls: the class (or a function); pairs: a predicate
    on (lens, digital); noop: the oracle's bytes equal the base row's; geom: output geometry rows, a function of pix returning
    (extra case keys, output length) on top of geometry A."""

    def __init__(self, name, group, case=None, add=0, remove=0, cls="general", pairs=None, noop=False, geom=None):
        self.name, self.group, self._case, self._add, self._remove, self._cls = name, group, case or {}, add, remove, cls
        self._pairs, self.noop, self.geom = pairs, noop, geom

    @staticmethod
    def _v(x, lens, digital, pix):
        return x(lens, digital, pix) if callable(x) else x

    def case(self, lens, digital, pix):
        return self._v(self._case, lens, digital, pix)

    def add(self, lens, digital, pix):
        return self._v(self._add, lens, digital, pix)

    def remove(self, lens, digital, pix):
        return self._v(self._remove, lens, digital, pix)

    def cls(self, lens, digital, pix):
        return self._v(self._cls, lens, digital, pix)

    def applies(self, lens, digital):
        return self._pairs is None or self._pairs(lens, digital)

    def __repr__(self):
        return self.name


# ---- the rows -------------------------------------------------------------------------------------------------------------------
def _pixel_limit(lens, digital, pix):
    sdt = abi.PIXEL_TYPES[pix][2]
    return dict(params=dict(pixel_value_limit={"u1": 200.0, "u2": 60000.0}.get(sdt, 0.7)))


def _more_rows(n):
    """A table of n rows more than the readout length: the extra rows carry a strongly different rotation, so a kernel that reads one
    of them renders other bytes."""
    def hook(m):
        d = m[-1] - m[-2]
        return np.concatenate([m] + [m[-1:] + d * (40.0 * (i + 1)) for i in range(n)])
    return hook


def _misaligned(which):
    """Input or output pointer one scalar past a 64-byte boundary: whole-pixel vector access is then illegal unless the pixel's
    alignment is one scalar (F_SRC_VEC / F_DST_VEC); 8-byte source words never are (F_SRC_VEC8)."""
    def extra(lens, digital, pix):
        return {which + "_offset": np.dtype(abi.PIXEL_TYPES[pix][2]).itemsize}

    def lost(lens, digital, pix):
        sb = np.dtype(abi.PIXEL_TYPES[pix][2]).itemsize
        _, align = _bpp_align(pix)
        if which == "src":
            return F["F_SRC_VEC8"] | (F["F_SRC_VEC"] if sb % align else 0)
        return F["F_DST_VEC"] if sb % align else 0

    def cls(lens, digital, pix):
        sb = np.dtype(abi.PIXEL_TYPES[pix][2]).itemsize
        return "general" if sb % _bpp_align(pix)[1] else "packed"
    return extra, lost, cls


def _out_geometry(pix, cut=None, wide=False, scaled=False):
    """Identity output maps (the packed kernel's integer prologue) with an output rect inside a larger buffer: 61 x 37 at (5, 2) in a
    70 x 41 buffer (written columns [x0, x1) = [5, 66)), or (wide) 75 x 43 at the origin of an 80-pixel wide buffer ([0, 75)).
    scaled: the 61 x 37 output drawn into a 58 x 35 rect (no longer the identity: no integer prologue).
    cut: None (the whole buffer), ("px", row, col) (the buffer ends part-way through pixel col of that row) or ("rows", n) (it ends at
    the end of row n - 1, stride padding included)."""
    bpp, align = _bpp_align(pix)
    base = geometries(pix)[0][1]
    if wide:
        ow, oh, obw, obh, rect = W, H, 80, H, (0, 0, W, H)
    else:
        ow, oh, obw, obh, rect = 61, 37, 70, 41, ((5, 2, 58, 35) if scaled else (5, 2, 61, 37))
    lcm8 = max(8, align)
    pad = (-(obw * bpp)) % lcm8 + lcm8
    ostride = obw * bpp + pad
    case = dict(base, ow=ow, oh=oh, out_size=(obw, obh), out_rect=rect, out_stride_pad=pad)
    if cut is None:
        n = obh * ostride
    elif cut[0] == "px":
        n = cut[1] * ostride + cut[2] * bpp + bpp // 2
    else:
        n = cut[1] * ostride
    return case, n


_mis_src, _mis_dst = _misaligned("src"), _misaligned("dst")
FIX, FILL, FBINV, DIGI = abi.FLAG_FIX_COLOR_RANGE, abi.FLAG_FILL_WITH_BACKGROUND, abi.FLAG_FRAMEBUFFER_INVERTED, abi.FLAG_HAS_DIGITAL_LENS
# a principal point near the bottom (right) edge: the last rows of the table (the last columns with horizontal readout) are then picked
# on every lens, also on insta360 whose synthetic profile keeps a fov 1.3 frame away from them
LOW_C, RIGHT_C, FAR_RIGHT_C = [W / 2.0, 38.0], [70.0, H / 2.0], [80.0, H / 2.0]
NOOP_GENERAL = lambda lens, digital, pix: "general" if lens in NOOP_LENSES else "packed"

ROWS = [
    # general-only features: the general kernel's run-time branches
    Row("horizontal-readout", "general", dict(horizontal_rs=True), bits("F_HRS")),
    Row("r_limit", "general", dict(fov=2.5, params=dict(r_limit=0.9)), bits("F_RLIMIT")),
    Row("refraction", "general", dict(params=dict(light_refraction_coefficient=1.33)), bits("F_REFRACT")),
    Row("refraction+lens-correction", "general", dict(params=dict(light_refraction_coefficient=1.33, lens_correction_amount=0.6)), bits("F_REFRACT", "F_LCA")),
    Row("lens-correction-0.35", "general", dict(params=dict(lens_correction_amount=0.35)), bits("F_LCA")),
    Row("lens-correction-0", "general", dict(params=dict(lens_correction_amount=0.0)), bits("F_LCA")),
    Row("stretch", "general", dict(params=dict(input_horizontal_stretch=1.3333, input_vertical_stretch=0.9)), bits("F_HSTRETCH", "F_VSTRETCH")),
    Row("horizontal-stretch", "general", dict(params=dict(input_horizontal_stretch=1.3333, input_vertical_stretch=1.0)), bits("F_HSTRETCH")),
    Row("input-rotation-90", "general", dict(params=dict(input_rotation=90.0)), bits("F_INROT")),
    Row("input-rotation--13.5+bg2", "general", dict(params=dict(input_rotation=-13.5, background_mode=2, background=BG)), bits("F_INROT", "F_BG2")),
    Row("translation3d", "general", dict(params=dict(translation3d=[0.5, -0.25, 0.002, 0.0])), bits("F_T3D")),
    Row("mesh-9", "general", dict(mesh=True, mesh_n=9), bits("F_MESH")),
    Row("mesh-7", "general", dict(mesh=True, mesh_n=7), bits("F_MESH")),
    Row("mesh+fpd", "general", dict(mesh=True, fpd=True), bits("F_MESH")),
    Row("mesh+fpd+fb-inverted", "general", dict(mesh=True, fpd=True, flags=FBINV), bits("F_MESH", "F_FB_INV")),
    Row("everything", "general", dict(horizontal_rs=True, mesh=True, fpd=True, flags=FBINV | FIX,
                                      params=dict(r_limit=1.6, light_refraction_coefficient=1.2, lens_correction_amount=0.6, input_horizontal_stretch=1.1,
                                                  input_vertical_stretch=0.95, input_rotation=-13.5, background_mode=3, background_margin=0.1,
                                                  background_margin_feather=0.15, background=BG, translation3d=[0.1, -0.05, 0.002, 0.0])),
        bits("F_HRS", "F_RLIMIT", "F_REFRACT", "F_MESH", "F_HSTRETCH", "F_VSTRETCH", "F_LCA", "F_INROT", "F_BG3", "F_FIXRANGE", "F_FB_INV", "F_T3D")),
    # general-only features that act on the pixel values: also every pixel type on PIXEL_PAIRS
    Row("background-1", "pixel", dict(fov=2.5, params=dict(background_mode=1, background=BG)), bits("F_BG1")),
    Row("background-2", "pixel", dict(fov=2.5, params=dict(background_mode=2, background=BG)), bits("F_BG2")),
    Row("background-3", "pixel", dict(fov=2.5, params=dict(background_mode=3, background_margin=0.1, background_margin_feather=0.15, background=BG)), bits("F_BG3")),
    Row("fix-range-plane-0", "pixel", dict(flags=FIX), bits("F_FIXRANGE")),
    Row("fix-range-plane-1", "pixel", dict(flags=FIX, params=dict(plane_index=1)), bits("F_FIXRANGE"), bits("F_IS_Y")),
    Row("fill-with-background", "pixel", dict(flags=FILL, params=dict(background=[0.3, 0.6, 0.9, 1.0])), bits("F_FILLBG")),
    Row("pixel-value-limit", "pixel", _pixel_limit, bits("F_PIXLIMIT")),
    # lens coefficients: the early-out of the four models that have one (fisheye / sony: k0..k3, generic: all twelve, gopro: k1)
    Row("k-all-zero", "lens", dict(params=dict(k=[0.0] * 12)),
        lambda lens, digital, pix: (F["F_LENS_NOOP"] if lens in NOOP_LENSES else 0) | (F["F_WILD"] if lens == "gopro" else 0), 0, NOOP_GENERAL),
    Row("sony-k0..k3-zero", "lens", dict(params=dict(k=[0.0, 0.0, 0.0, 0.0, 0.02, -0.004] + [0.0] * 6)), bits("F_LENS_NOOP"),
        pairs=lambda lens, digital: lens == "sony"),
    Row("generic-k0..k10-zero", "lens", dict(params=dict(k=[0.0] * 11 + [0.0004])), 0, cls="packed", pairs=lambda lens, digital: lens == "generic_polynomial"),
    Row("gopro-k1-zero", "lens", dict(params=dict(k=[0.0, 0.0, 0.01, 0.12, -0.03, 0.02, 0.005] + [0.0] * 5)), bits("F_LENS_NOOP", "F_WILD"),
        pairs=lambda lens, digital: lens == "gopro"),
    Row("fisheye-k0..k3-zero", "lens", dict(params=dict(k=[0.0, 0.0, 0.0, 0.0, 0.05, -0.02] + [0.0] * 6)), bits("F_LENS_NOOP"),
        pairs=lambda lens, digital: lens == "opencv_fisheye"),
    # a digital-lens context rendering a frame without its digital lens (flag bit 2 clear)
    Row("digital-flag-clear", "digital", dict(clear_flags=DIGI), 0, bits("F_DIGITAL"), pairs=lambda lens, digital: digital is not None),
    Row("digital-flag-clear+lens-correction", "digital", dict(clear_flags=DIGI, params=dict(lens_correction_amount=0.5)), bits("F_LCA"), bits("F_DIGITAL"),
        pairs=lambda lens, digital: digital is not None),
    # no-ops: the oracle's bytes equal the base row's
    Row("stretch-0.001", "noop", dict(params=dict(input_horizontal_stretch=0.001, input_vertical_stretch=0.001)), cls="packed", noop=True),
    Row("stretch-1.0", "noop", dict(params=dict(input_horizontal_stretch=1.0, input_vertical_stretch=0.0)), cls="packed", noop=True),
    Row("translation3d-negative-zero", "noop", dict(params=dict(translation3d=[-0.0, -0.0, -0.0, 0.0])), cls="packed", noop=True),
    Row("fb-inverted-without-mesh", "noop", dict(flags=FBINV), bits("F_FB_INV"), noop=True),
    # matrix tables
    Row("matrix-count-2", "table", dict(matrix_hook=lambda m: m[:2]), cls="packed"),
    Row("matrix-count-3", "table", dict(matrix_hook=lambda m: m[:3]), cls="packed"),
    Row("matrix-count-h-1", "table", dict(matrix_hook=lambda m: m[:-1], params=dict(c=LOW_C)), cls="packed"),
    Row("matrix-count-h+1", "table", dict(matrix_hook=_more_rows(1), params=dict(c=LOW_C)), cls="packed"),
    Row("matrix-count-h+9", "table", dict(matrix_hook=_more_rows(9), params=dict(c=LOW_C)), cls="packed"),
    Row("horizontal-readout-w-1", "table", dict(horizontal_rs=True, matrix_hook=lambda m: m[:-1], params=dict(c=RIGHT_C)), bits("F_HRS")),
    Row("horizontal-readout-w+1", "table", dict(horizontal_rs=True, matrix_hook=_more_rows(1), params=dict(c=FAR_RIGHT_C)), bits("F_HRS")),
    Row("rolling-shutter-off", "table", dict(rs=False), 0, bits("F_RS"), cls="packed"),
    Row("ibis", "table", dict(ibis=True), cls="guarded"),
    Row("translation2d", "table", dict(params=dict(translation2d=[4.5, -3.25])), cls="packed"),
    Row("wild-principal-point", "table", dict(params=dict(c=[0.0, H / 2.0])), bits("F_WILD"), cls="lean"),
    # output geometry (on top of geometry A's input)
    Row("out-rect-offset", "geometry", cls="packed", geom=lambda pix: _out_geometry(pix)),
    Row("out-rect-scaled", "geometry", remove=bits("F_INTPRO"), cls="packed", geom=lambda pix: _out_geometry(pix, scaled=True)),
    Row("out-buffer-wider", "geometry", cls="packed", geom=lambda pix: _out_geometry(pix, wide=True)),
    Row("cut-left-of-x0", "geometry", cls="packed", geom=lambda pix: _out_geometry(pix, ("px", 20, 3))),
    Row("cut-inside", "geometry", add=bits("F_SHORTROW"), cls="packed", geom=lambda pix: _out_geometry(pix, ("px", 20, 29))),
    Row("cut-right-of-x1", "geometry", cls="packed", geom=lambda pix: _out_geometry(pix, ("px", 20, 68))),
    Row("cut-right-of-x1-wide", "geometry", cls="packed", geom=lambda pix: _out_geometry(pix, ("px", 20, 77), wide=True)),
    Row("cut-at-row-end", "geometry", cls="packed", geom=lambda pix: _out_geometry(pix, ("rows", 21))),
    Row("src-misaligned", "geometry", _mis_src[0], 0, _mis_src[1], _mis_src[2], noop=True),
    Row("dst-misaligned", "geometry", _mis_dst[0], 0, _mis_dst[1], _mis_dst[2], noop=True),
]
BASE = Row("base", "base", cls="packed")
BY_NAME = {r.name: r for r in ROWS}
GENERAL_GROUPS = ("general", "pixel")


def rows_of(*groups):
    return [r for r in ROWS if r.group in groups]


def cell_case(row, lens, digital, pix, geom="A/stride8"):
    """(case, output length) of a cell: the row's override on the base frame in the named geometry of test_kernel_matrix (fov 1.3),
    or, for output geometry rows, on geometry A's input."""
    if row.geom:
        case, out_len = row.geom(pix)
        return dict(case, fov=1.3), out_len
    for name, case, out_len in geometries(pix):
        if name == geom:
            return dict(dict(case, fov=1.3), **row.case(lens, digital, pix)), out_len
    raise KeyError(geom)


def row_geoms(row):
    """The geometries a row renders in: general-only rows also in geometry B (non-identity maps, short output)."""
    return ("A/stride8", "B/ends-mid-row") if row.group in GENERAL_GROUPS else ("A/stride8",)


def expected_code(cls, mode):
    """The gf_cuda_plan code of a row's class under one variant of MODES."""
    _, switch, interp, tables, code = mode
    two = code & 0x10
    if cls == "general":
        return two
    if cls == "lean":
        return two | (0 if switch == "GF_DISABLE_LEAN" else 1)
    if cls == "guarded":
        return two | min(code & 0xF, 2)
    return code


def _mesh_len(case, pix, lens, digital):
    return cases.build(dict(case, pix=pix, lens=lens, digital=digital))[3].size if case.get("mesh") else 0


def features(case, pix, lens, digital, interp, out_len, tables):
    """(gf_cuda_plan_features code, feature word) of a cell; tables: "host" (the host scan's verdict), "device" (non-zero), or an int."""
    p, src, m, dst = build(case, pix, lens, digital, interp, out_len)
    bufs = descs(case, p, src, dst, out_len)
    lib = g.load_library()
    flags = lib.gf_table_flags_host(m.ctypes.data, m.shape[0]) if tables == "host" else (1 if tables == "device" else tables)
    i, o = bufs.input.to_c(), bufs.output.to_c()
    feat = C.c_uint32(0xFFFFFFFF)
    code = lib.gf_cuda_plan_features(C.byref(p), abi.PIXEL_TYPES[pix][0], abi.LENS[lens], abi.LENS[digital] if digital else 0,
                                     C.byref(i), C.byref(o), _mesh_len(case, pix, lens, digital), flags, 1, C.byref(feat))
    return code, feat.value


def oracle_bytes(row, lens, digital, pix):
    case, out_len = cell_case(row, lens, digital, pix)
    p, src, m, dst = build(case, pix, lens, digital, "Bilinear", out_len)
    mesh = cases.build(dict(case, pix=pix, lens=lens, digital=digital))[3] if case.get("mesh") else None
    want = dst[:out_len].copy()
    assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
    return want


def cells(rows, pairs, pixel_types):
    for row in rows:
        for lens, digital in pairs:
            if row.applies(lens, digital):
                for pix in pixel_types:
                    yield row, lens, digital, pix


# ---- the feature word, without a GPU ---------------------------------------------------------------------------------------------
def _enum():
    text = open(os.path.join(ROOT, "gyroflow_b200", "csrc", "warp_kernel.cuh")).read()
    body = re.search(r"// feature bits.*?enum\s*:\s*uint32_t\s*\{(.*?)\};", text, re.S).group(1)
    enum = {n: 1 << int(s) for n, s in re.findall(r"(F_[A-Z0-9_]+)\s*=\s*1u\s*<<\s*(\d+)", body)}
    go = re.search(r"F_GENERAL_ONLY\s*=\s*(.*?);", text, re.S).group(1)
    return enum, [n.strip() for n in go.split("|")]


def test_abi_mirrors_the_feature_enum():
    """abi.F and abi.F_GENERAL_ONLY are the enum and the mask of warp_kernel.cuh, bit for bit."""
    enum, general_only = _enum()
    assert len(enum) >= 27 and enum == abi.F
    mask = 0
    for n in general_only:
        mask |= enum[n]
    assert mask == abi.F_GENERAL_ONLY


def test_plan_features_agrees_with_plan():
    """gf_cuda_plan_features returns gf_cuda_plan's code, and a word equal to the bits fill_uniforms computes (no stray bits)."""
    lib = g.load_library()
    allbits = 0
    for v in abi.F.values():
        allbits |= v
    for lens, digital in PIXEL_PAIRS:
        for tables in ("host", "device"):
            case, out_len = cell_case(BASE, lens, digital, "RGBA8")
            p, src, m, dst = build(case, "RGBA8", lens, digital, "Bilinear", out_len)
            bufs = descs(case, p, src, dst, out_len)
            from tests.test_kernel_matrix import plan
            flags = lib.gf_table_flags_host(m.ctypes.data, m.shape[0]) if tables == "host" else 1
            code, feat = features(case, "RGBA8", lens, digital, "Bilinear", out_len, tables)
            assert code == plan(p, "RGBA8", lens, digital, bufs, flags) and feat & ~allbits == 0
    i = abi.BufferDesc()
    assert lib.gf_cuda_plan_features(None, 0, 1, 0, C.byref(i), C.byref(i), 0, 0, 1, None) == -1


def _declared(row, lens, digital, pix):
    return row.add(lens, digital, pix), row.remove(lens, digital, pix)


def test_rows_set_exactly_their_bits(monkeypatch):
    """Every row, on every pair and pixel type it runs on, in every geometry it renders in: the word differs from the base frame's word
    (same pair, pixel type and geometry) in exactly the declared bits, F_FILTER aside, which is set iff the packed kernel renders a
    fisheye frame without a digital lens, with rolling shutter and trusted tables.  Together the rows change every bit of the enum."""
    set_switch(monkeypatch, None)
    changed, checked = 0, 0
    for row, lens, digital, pix in cells(ROWS, library_pairs(), GEN_PIX):
        for geom in row_geoms(row):
            case, out_len = cell_case(row, lens, digital, pix, geom)
            code, word = features(case, pix, lens, digital, "Bilinear", out_len, "host")
            bcase, bout = cell_case(BASE, lens, digital, pix, geom)
            _, base = features(bcase, pix, lens, digital, "Bilinear", bout, "host")
            add, remove = _declared(row, lens, digital, pix)
            where = (row, lens, digital, pix, geom, hex(word), hex(base))
            assert (word ^ base) & ~F["F_FILTER"] == add | remove, where
            assert word & add == add and word & remove == 0, where
            filt = (code & 0xF) == 3 and lens == "opencv_fisheye" and digital is None and bool(word & F["F_RS"])
            assert bool(word & F["F_FILTER"]) == filt, where
            changed |= word ^ base
            checked += 1
    missing = [n for n, v in F.items() if not changed & v]
    assert not missing, "no row changes %s" % missing
    assert checked > 1500, checked


def test_plan_codes(monkeypatch):
    """gf_cuda_plan for every (row, pair, pixel type, geometry) under every variant of MODES: the code the row's class predicts."""
    lib = g.load_library()
    checked = set()
    for row, lens, digital, pix in cells(ROWS, library_pairs(), GEN_PIX):
        cls = row.cls(lens, digital, pix)
        for geom in row_geoms(row):
            case, out_len = cell_case(row, lens, digital, pix, geom)
            for interp in ("Bilinear", "Lanczos4"):
                p, src, m, dst = build(case, pix, lens, digital, interp, out_len)
                bufs = descs(case, p, src, dst, out_len)
                host_flags = lib.gf_table_flags_host(m.ctypes.data, m.shape[0])
                assert (host_flags != 0) == (cls == "guarded"), (row, lens, digital, pix)
                ml = _mesh_len(case, pix, lens, digital)
                from tests.test_kernel_matrix import plan
                for mode in MODES:
                    if mode[2] != interp:
                        continue
                    set_switch(monkeypatch, mode[1])
                    got = plan(p, pix, lens, digital, bufs, host_flags if mode[3] == "host" else 1, ml)
                    assert got == expected_code(cls, mode), (row, lens, digital, pix, geom, mode[0], got, expected_code(cls, mode))
                    checked.add((row.name, lens, digital, pix, mode[0]))
    assert len(checked) == sum(1 for _ in cells(ROWS, library_pairs(), GEN_PIX)) * len(MODES)


def test_rows_change_the_output():
    """Non-vacuity: on every pair and pixel type a row runs on, the oracle's bytes differ from the base row's; the declared no-ops
    equal them byte for byte."""
    for row, lens, digital, pix in cells(ROWS, library_pairs(), GEN_PIX):
        got, base = oracle_bytes(row, lens, digital, pix), oracle_bytes(BASE, lens, digital, pix)
        same = got.shape == base.shape and np.array_equal(got, base)
        assert same == row.noop, (row, lens, digital, pix, "no-op row changed the output" if row.noop else "row does not change the output")
        if "matrix_hook" in row.case(lens, digital, pix):       # the table's length itself matters, not just the row's other keys
            full = Row(row.name + " with the readout-length table", row.group, {k: v for k, v in row.case(lens, digital, pix).items() if k != "matrix_hook"})
            assert not np.array_equal(got, oracle_bytes(full, lens, digital, pix)), (row, lens, digital, pix, "the table's length changes nothing")


# rows whose semantics no other test restates, on a few pairs: the restatement must produce the oracle's bytes
RESTATED = [("translation3d", "opencv_fisheye", None), ("translation3d", "sony", "digital_stretch"),
            ("sony-k0..k3-zero", "sony", None), ("generic-k0..k10-zero", "generic_polynomial", None), ("gopro-k1-zero", "gopro", None),
            ("fisheye-k0..k3-zero", "opencv_fisheye", None), ("k-all-zero", "opencv_fisheye", "gopro_superview"), ("k-all-zero", "poly5", None),
            ("digital-flag-clear", "opencv_fisheye", "gopro_hyperview"), ("digital-flag-clear+lens-correction", "poly3", "digital_stretch"),
            ("digital-flag-clear+lens-correction", "gopro", "gopro_warp"),
            ("matrix-count-2", "opencv_fisheye", None), ("matrix-count-h-1", "opencv_fisheye", None), ("matrix-count-h+1", "ptlens", None),
            ("horizontal-readout-w-1", "opencv_fisheye", None), ("horizontal-readout-w+1", "opencv_fisheye", None),
            ("stretch-0.001", "opencv_fisheye", None), ("stretch-1.0", "insta360", None), ("horizontal-stretch", "opencv_standard", None)]


@pytest.mark.parametrize("name,lens,digital", RESTATED)
def test_restatement_agrees(name, lens, digital):
    """The oracle and tests/np_restatement.py agree byte for byte on the row (a small 36 x 20 frame, fov 1.3, rolling shutter on)."""
    from tests import np_restatement
    case = dict(dict(w=36, h=20, fov=1.3, pix="RGBA8", lens=lens, digital=digital), **BY_NAME[name].case(lens, digital, "RGBA8"))
    p, src, m, mesh, dst0, pix, lens, digital = cases.build(case)
    want = dst0.copy()
    assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
    got = dst0.copy()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        np_restatement.undistort_image(src, got, p, m, lens=lens, sdt=np.uint8, digital=digital, mesh=mesh)
    assert np.array_equal(got, want), (name, lens, digital, int((got != want).sum()))


# ---- the GPU matrix --------------------------------------------------------------------------------------------------------------
def expected_launches(code, interp, case, pix, lens, digital, out_len, tables):
    """One launch (bilinear), two (coordinate + sampling pass) or four (EWA), plus the tail launch of the packed kernel's filtered
    pre-pass when the plan runs it: the word's F_FILTER, with device tables as trusted as the verdict word they carry."""
    n = 1 if interp == "Bilinear" else (4 if interp.startswith("EWA") else 2)
    if (code & 0xF) >= 2 and lens == "opencv_fisheye" and digital is None:
        _, word = features(case, pix, lens, digital, interp, out_len, 0 if tables == "device" else "host")
        n += 1 if word & F["F_FILTER"] else 0
    return n


def run_rows(request, monkeypatch, rows, pairs, pixel_types, modes, kinds_of, label, geoms=None):
    """Render every (row, pair, pixel type, geometry, variant) cell with every buffer kind of kinds_of(geometry); report the count, the
    time and the failing cells; fail on the first bad render.  Returns the number of cells."""
    t0 = time.perf_counter()
    n_cells, renders, bad, bad_cells = 0, 0, [], set()
    for row, lens, digital, pix in cells(rows, pairs, pixel_types):
        bpp, _ = _bpp_align(pix)
        cls = row.cls(lens, digital, pix)
        for geom in geoms or row_geoms(row):
            case, out_len = cell_case(row, lens, digital, pix, geom)
            for mode in modes:
                set_switch(monkeypatch, mode[1])
                _, _, interp, tables, _ = mode
                cell = (row.name, lens, digital, pix, geom, mode[0])
                # HOST buffers are staged into the library's own (aligned) device buffers: only DEVICE buffers reach the kernel misaligned
                kinds = ("device",) if case.get("src_offset") or case.get("dst_offset") else kinds_of(geom)
                want, outs, code = render(case, pix, lens, digital, interp, tables, out_len, kinds)
                assert code == expected_code(cls, mode), (cell, code)
                launches_want = expected_launches(code, interp, case, pix, lens, digital, out_len, tables)
                for kind, got, launches in outs:
                    renders += 1
                    where = "%s %s" % (cell, kind)
                    assert launches == launches_want, (where, launches, launches_want)
                    if not np.array_equal(got[out_len:], np.full(GUARD, 0xA5, np.uint8)):
                        bad.append("%s: wrote past the end of the output" % where); bad_cells.add(cell)
                    elif not np.array_equal(got[:out_len], want):
                        stride = cases.build(dict(case, pix=pix, lens=lens, digital=digital))[0].output_stride
                        bad.append("%s: %d bytes differ, first at %s" % (where, int((got[:out_len] != want).sum()), _first_bad(want, got[:out_len], stride, bpp)))
                        bad_cells.add(cell)
                n_cells += 1
    report(request, "%s: %d cells, %d renders, %d failing renders in %d cells, %.1f s" %
           (label, n_cells, renders, len(bad), len(bad_cells), time.perf_counter() - t0))
    for c in sorted(bad_cells, key=str)[:64]:
        report(request, "  failing cell: %s" % (c,))
    assert not bad, "%d failing renders; first: %s" % (len(bad), bad[0])
    return n_cells


def _n_cells(rows, pairs, pixel_types, n_modes, geoms=None):
    return sum(len(geoms or row_geoms(r)) for r, _, _, _ in cells(rows, pairs, pixel_types)) * n_modes


def _a_both_b_host(geom):
    return ("host", "device") if geom.startswith("A") else ("host",)


@pytest.mark.gpu
def test_general_rows(request, monkeypatch):
    """General-only rows on every pair x {RGBA8, Luma16, RGBAf}: fused bilinear and the Lanczos4 coordinate pass of the general kernel,
    geometry A (HOST and DEVICE) and geometry B (HOST)."""
    rows, pairs = rows_of(*GENERAL_GROUPS), library_pairs()
    n = run_rows(request, monkeypatch, rows, pairs, GEN_PIX, GEN_MODES, _a_both_b_host, "test_general_rows")
    assert n == _n_cells(rows, pairs, GEN_PIX, 2) == len(rows) * 21 * 3 * 2 * 2


@pytest.mark.gpu
def test_pixel_rows_every_pixel_type(request, monkeypatch):
    """Rows that act on pixel values (background modes, fix range, fill, pixel_value_limit) in all 13 pixel types on three pairs."""
    rows = rows_of("pixel")
    n = run_rows(request, monkeypatch, rows, PIXEL_PAIRS, PIXEL_TYPES, GEN_MODES, lambda geom: ("host",), "test_pixel_rows_every_pixel_type")
    assert n == len(rows) * 3 * 13 * 2 * 2


@pytest.mark.gpu
def test_general_rows_ewa(request, monkeypatch):
    """General-only rows with EWA (three coordinate maps, four launches) on three pairs in RGBA8 and RGBAf.  Not r_limit: a Jacobian
    probe beyond the limit next to a valid centre gives a footprint past the kernel's 2^22-tap guard, which renders background where
    the reference (and the oracle) sum the whole box: the footprint guard documented in warp_kernel.cuh."""
    rows = [r for r in rows_of(*GENERAL_GROUPS) if r.name != "r_limit"]
    n = run_rows(request, monkeypatch, rows, PIXEL_PAIRS, ["RGBA8", "RGBAf"], [EWA_MODE], lambda geom: ("host",), "test_general_rows_ewa",
                 geoms=("A/stride8",))
    assert n == len(rows) * 3 * 2


@pytest.mark.gpu
def test_lens_digital_and_noop_rows(request, monkeypatch):
    """Lens-coefficient, cleared digital flag and no-op rows: every pair they apply to x {RGBA8, Luma16, RGBAf} x all 7 variants."""
    rows, pairs = rows_of("lens", "digital", "noop"), library_pairs()
    n = run_rows(request, monkeypatch, rows, pairs, GEN_PIX, MODES, lambda geom: ("host", "device"), "test_lens_digital_and_noop_rows")
    # k all zero: 21 pairs; sony, generic, gopro partial zeros: 2 pairs each; fisheye: 5; cleared digital flag: the 12 digital pairs
    assert n == _n_cells(rows, pairs, GEN_PIX, 7) == (21 + 2 + 2 + 2 + 5 + 12 * 2 + 4 * 21) * 3 * 7


@pytest.mark.gpu
def test_row_tables(request, monkeypatch):
    """Matrix tables of 2, 3, h - 1, h + 1 and h + 9 rows, horizontal readout with w - 1 and w + 1, rolling shutter off, IBIS rows,
    translation2d and F_WILD: every pair x {RGBA8, Luma16, RGBAf} x all 7 variants, HOST and DEVICE outputs."""
    rows, pairs = rows_of("table"), library_pairs()
    n = run_rows(request, monkeypatch, rows, pairs, GEN_PIX, MODES, lambda geom: ("host", "device"), "test_row_tables")
    assert n == len(rows) * 21 * 3 * 7


@pytest.mark.gpu
def test_output_geometry(request, monkeypatch):
    """Identity output maps with an offset output rect and a buffer wider than the output, buffers cut left of x0, inside [x0, x1),
    right of x1 and at a row end, and misaligned input / output pointers: every pair x {RGBA8, Luma16, RGBAf} x all 7 variants, HOST
    and DEVICE outputs (HOST outputs switch full_cover off and upload the buffer first)."""
    rows, pairs = rows_of("geometry"), library_pairs()
    n = run_rows(request, monkeypatch, rows, pairs, GEN_PIX, MODES, lambda geom: ("host", "device"), "test_output_geometry")
    assert n == len(rows) * 21 * 3 * 7


@pytest.mark.gpu
def test_general_rows_fused_planes(request, monkeypatch):
    """General-only rows as a fused two-plane frame (gf_cuda_undistort_planes_dev: one coordinate pass, one sampling pass per plane) on
    three pairs in RGBA8 and Luma16, each plane byte for byte against its own oracle run, guard bytes untouched."""
    import torch
    set_switch(monkeypatch, None)
    t0, n, bad = time.perf_counter(), 0, []
    rows = rows_of(*GENERAL_GROUPS)
    for row, lens, digital, pix in cells(rows, PIXEL_PAIRS, ["RGBA8", "Luma16"]):
        case, out_len = cell_case(row, lens, digital, pix)
        planes = []
        for i in range(2):
            p, src, m, dst = build(dict(case, frame=i), pix, lens, digital, "Bilinear", out_len)
            p = p.copy(); p.plane_index = i
            p.background[:] = [0.1 * (i + 1), 0.5, 0.25, 1.0]
            mesh = cases.build(dict(case, pix=pix, lens=lens, digital=digital))[3] if case.get("mesh") else None
            want = dst[:out_len].copy()
            assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
            planes.append((p, src, m, dst, mesh, want))
        p0, _, m, _, mesh, _ = planes[0]
        tsrc = [torch.from_numpy(s.copy()).cuda() for _, s, _, _, _, _ in planes]
        tdst = [torch.from_numpy(d.copy()).cuda() for _, _, _, d, _, _ in planes]
        bufs = [descs(case, p, s, d, out_len) for (p, _, _, _, _, _), s, d in zip(planes, tsrc, tdst)]
        tm = torch.from_numpy(m).cuda()
        tmesh = torch.from_numpy(mesh).cuda() if mesh is not None else None
        ctx = g.CudaWrapper.new(p0, pix, lens, digital, bufs[0])
        try:
            l0 = ctx.launch_count
            ctx.undistort_planes_dev(bufs, [pl[0] for pl in planes], tm.data_ptr(), m.shape[0], tmesh.data_ptr() if tmesh is not None else 0,
                                     0 if mesh is None else mesh.size)
            ctx.synchronize()
            launches = ctx.launch_count - l0
        finally:
            ctx.close()
        assert launches == 3, (row, lens, digital, pix, launches)
        for i, (pl, d) in enumerate(zip(planes, tdst)):
            got = d.cpu().numpy()
            if not np.array_equal(got[out_len:], np.full(GUARD, 0xA5, np.uint8)):
                bad.append("%s plane %d: wrote past the end of the output" % ((row.name, lens, digital, pix), i))
            elif not np.array_equal(got[:out_len], pl[5]):
                bad.append("%s plane %d: %d bytes differ" % ((row.name, lens, digital, pix), i, int((got[:out_len] != pl[5]).sum())))
        n += 1
    report(request, "test_general_rows_fused_planes: %d frames of 2 planes, %d failing planes, %.1f s" % (n, len(bad), time.perf_counter() - t0))
    assert not bad, "%d failing planes; first: %s" % (len(bad), bad[0])
    assert n == len(rows) * 3 * 2
