"""Every compiled warp kernel against the CPU oracle, cell by cell.

A cell is one (lens pair, pixel type, kernel variant).  The pairs are the ones the library compiles (the 21 the reference
pre-compiles), the pixel types all 13, and the variants the nine ways a frame can be rendered (MODES): the packed kernel on its
trusted and on its guarded path, the lean and the general kernel, the three coordinate passes of the two-pass path, and the lean and
general coordinate passes with EWA's two Jacobian probe passes.  A switch
(GF_DISABLE_X2, GF_DISABLE_LEAN) or the tables' provenance selects the variant; gf_cuda_plan, which shares the planner with the
rendering call, says which one a frame takes.

test_plan_matrix checks that choice for every cell without a GPU.  The GPU tests render every cell, in two geometries, byte for byte
against oracle_lib.undistort_image, and count what they rendered so that no cell can drop out silently.  test_edge_values feeds
float and 16-bit content at the edges of the value domain (synth.edge_frame) through every variant and resampler.
"""
import ctypes as C
import time

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi
from tests import cases, oracle_lib

# the (lens, digital lens) pairs the reference pre-compiles (qt_gpu/compiled/compile_shaders.sh:6-27)
REFERENCE_PAIRS = [("opencv_fisheye", d) for d in (None, "gopro_superview", "gopro6_superview", "gopro_hyperview", "digital_stretch")] + \
                  [("gopro", None), ("gopro", "gopro_warp")] + \
                  [(l, d) for l in ("opencv_standard", "poly3", "poly5", "ptlens", "insta360", "sony", "generic_polynomial") for d in (None, "digital_stretch")]
PIXEL_TYPES = sorted(abi.PIXEL_TYPES)
SWITCHES = ("GF_DISABLE_X2", "GF_DISABLE_LEAN", "GF_DISABLE_FILTER")

# (variant, switch, resampler, tables, gf_cuda_plan code).  Host tables are scanned on the host (tame: verdict 0, trusted path);
# device tables without a verdict word take the guarded path.  Every pair has a packed form for every pixel layout, and the
# geometries below keep pixel alignment, so no cell is an exception to its mode's code.
MODES = [
    ("packed", None, "Bilinear", "host", 3),
    ("packed-guarded", None, "Bilinear", "device", 2),
    ("lean", "GF_DISABLE_X2", "Bilinear", "host", 1),
    ("general", "GF_DISABLE_LEAN", "Bilinear", "host", 0),
    ("packed-coords", None, "Lanczos4", "host", 0x13),
    ("lean-coords", "GF_DISABLE_X2", "Lanczos4", "host", 0x11),
    ("general-coords", "GF_DISABLE_LEAN", "Lanczos4", "host", 0x10),
    # EWA: three coordinate maps (the pixel and its two Jacobian probes) and no packed form.  The kernel reads the filter only as
    # KernelParams::ewa_coeffs, so the two variants take two different filters rather than all four each.
    ("lean-ewa", None, "EWA: RobidouxSharp", "host", 0x11),
    ("general-ewa", "GF_DISABLE_LEAN", "EWA: Catmull-Rom", "host", 0x10),
]
# (lens, digital, geometry) cells EWA cannot be compared in: in geometry B, next to its NaN centres, (opencv_fisheye, gopro_hyperview)
# has written pixels whose Jacobian probes give footprints past the kernel's 2^22-tap guard, up to a saturated i32 box that the oracle
# would sum ~1e19 taps for (test_ewa_resampler.test_geometry_b_footprints pins both)
EWA_UNCOMPARABLE = {("opencv_fisheye", "gopro_hyperview", "B")}
W, H = 75, 43          # not a multiple of the 32-wide block nor of the packed kernel's 8-row tile: a lone last row is left over
CUT = 29                # the short output buffers end inside this pixel of the last row (at its first byte for 1-byte pixels)
GUARD = 2048            # bytes after the output's described length that must stay untouched (more than one output row)


def library_pairs():
    """Every (lens, digital lens) for which the library has a kernel in every pixel type."""
    lib = g.load_library()
    names = {v: k for k, v in abi.LENS.items()}
    out = []
    for lens in range(1, len(abi.LENS)):
        for dig in range(len(abi.LENS)):
            if all(lib.gf_combo_supported(abi.PIXEL_TYPES[p][0], lens, dig, abi.INTERP["Bilinear"]) for p in PIXEL_TYPES):
                out.append((names[lens], names[dig] if dig else None))
    return out


def _bpp_align(pix):
    _, count, sdt = abi.PIXEL_TYPES[pix]
    sb = np.dtype(sdt).itemsize
    bpp = count * sb
    return bpp, (bpp if bpp in (1, 2, 4, 8, 16) else sb)      # the alignment whole-pixel vector access needs


def geometries(pix):
    """(name, cases.build case, output length in bytes) of the two geometries: A in three forms, B in two.

    A: identity output maps (the packed kernel's integer prologue), input and output W x H with one padded stride.  Once with a
       stride that is a multiple of 8 (the Lanczos row window) and the whole buffer; then with a stride that is not (for 8- and
       16-byte pixels: another padded multiple) and a buffer that ends at the last pixel of the last row (HOST outputs: the
       full-cover 2-D copy back), then one that ends part-way through pixel 29 of the last row (X2Hot::full_rows / last_cols).
    B: non-identity maps: a source rect inside a larger input, an output of another size in an output rect inside a larger buffer
       that reaches its bottom-right corner (the last row is written up to its last pixel), fov 1.3 (background pixels); an output
       buffer that ends at that last pixel, then one that ends part-way through pixel 29 of the last row."""
    bpp, align = _bpp_align(pix)
    lcm8 = max(8, align)
    pad8 = -(-(W * bpp + 1) // lcm8) * lcm8 - W * bpp
    pad = align
    while (W * bpp + pad) % 8 == 0 and align < 8:
        pad += align
    if align >= 8:
        pad = pad8 + align
    stride = W * bpp + pad
    a = dict(w=W, h=H, stride_pad=pad)
    out = [("A/stride8", dict(w=W, h=H, stride_pad=pad8), H * (W * bpp + pad8)),
           ("A/ends-at-last-pixel", a, (H - 1) * stride + W * bpp),
           ("A/ends-mid-row", a, (H - 1) * stride + CUT * bpp + bpp // 2)]
    ow, oh = 61, 37
    obw, obh = 66, 41
    b = dict(w=W, h=H, ow=ow, oh=oh, fov=1.3, in_size=(83, 49), in_rect=(5, 4, 70, 40), out_size=(obw, obh), out_rect=(4, 3, obw - 4, obh - 3),
             stride_pad=align, out_stride_pad=2 * align)
    ostride = obw * bpp + 2 * align
    out.append(("B/ends-at-last-pixel", b, (obh - 1) * ostride + obw * bpp))
    out.append(("B/ends-mid-row", b, (obh - 1) * ostride + CUT * bpp + bpp // 2))
    return out


def _aligned(n, fill=0):
    raw = np.full(n + 64, fill, np.uint8)
    off = (-raw.ctypes.data) % 64
    return raw[off:off + n]


def build(case, pix, lens, digital, interp, out_len):
    """cases.build with 64-byte aligned buffers and an output of exactly out_len bytes (+ GUARD sentinel bytes after it).  The case
    keys src_offset / dst_offset start the input / output that many bytes past the 64-byte boundary instead."""
    p, src, m, mesh, dst0, _, _, _ = cases.build(dict(case, pix=pix, lens=lens, digital=digital, interp=interp))
    so, do = case.get("src_offset", 0), case.get("dst_offset", 0)
    a = _aligned(src.size + so)[so:]
    a[:] = src.reshape(-1)
    dst = _aligned(out_len + GUARD + do, 0xA5)[do:]
    return p, a, m, dst


def descs(case, p, src, dst, out_len):
    bw, bh = case.get("in_size", (case["w"], case["h"]))
    obw, obh = case.get("out_size", (case.get("ow", case["w"]), case.get("oh", case["h"])))
    if isinstance(src, np.ndarray):
        return g.Buffers(g.BufferDescription((bw, bh, p.stride), src), g.BufferDescription((obw, obh, p.output_stride), dst[:out_len]))
    return g.Buffers(g.BufferDescription((bw, bh, p.stride), src.data_ptr(), length=src.numel()),
                     g.BufferDescription((obw, obh, p.output_stride), dst.data_ptr(), length=out_len))


def plan(p, pix, lens, digital, bufs, table_flags, mesh_len=0):
    i, o = bufs.input.to_c(), bufs.output.to_c()
    return g.load_library().gf_cuda_plan(C.byref(p), abi.PIXEL_TYPES[pix][0], abi.LENS[lens], abi.LENS[digital] if digital else 0,
                                         C.byref(i), C.byref(o), mesh_len, table_flags, 1)


def set_switch(monkeypatch, switch):
    for s in SWITCHES:
        monkeypatch.delenv(s, raising=False)
    if switch:
        monkeypatch.setenv(switch, "1")


def expected_launches(code, interp, lens, digital):
    base = 1 if interp == "Bilinear" else (4 if interp.startswith("EWA") else 2)
    # the packed kernel's filtered rolling-shutter pre-pass (fisheye without a digital lens) adds the tail launch of its deferred pairs
    return base + (1 if (code & 0xF) >= 2 and lens == "opencv_fisheye" and digital is None else 0)


def report(request, msg):
    """Print past pytest's output capture, so that a passing run shows it too."""
    with request.getfixturevalue("capsys").disabled():
        print(msg)


# ---- the planner, without a GPU --------------------------------------------------------------------------------------------------
def test_library_pairs_are_the_reference_pairs():
    pairs = library_pairs()
    assert len(pairs) == 21 and sorted(pairs, key=str) == sorted(REFERENCE_PAIRS, key=str), pairs


def test_plan_matrix(monkeypatch):
    """gf_cuda_plan for every cell in every geometry the GPU matrix renders: 21 pairs x 13 pixel types x 9 variants."""
    lib = g.load_library()
    checked = set()
    for lens, digital in library_pairs():
        for pix in PIXEL_TYPES:
            for name, case, out_len in geometries(pix):
                for mode, switch, interp, tables, code in MODES:
                    set_switch(monkeypatch, switch)
                    p, src, m, dst = build(case, pix, lens, digital, interp, out_len)
                    flags = lib.gf_table_flags_host(m.ctypes.data, m.shape[0]) if tables == "host" else 1
                    assert tables == "device" or flags == 0, (lens, digital, pix, name)          # tame host tables: the trusted path
                    got = plan(p, pix, lens, digital, descs(case, p, src, dst, out_len), flags)
                    assert got == code, (lens, digital, pix, name, mode, got, code)
                    checked.add((lens, digital, pix, mode))
    assert len(checked) == 21 * 13 * 9


@pytest.mark.parametrize("pix", PIXEL_TYPES)
def test_short_buffers_end_in_written_pixels(pix):
    """The short output buffers cut the buffer where the CPU path writes: the pixel before each cut is written, the partial pixel at
    the cut is not (so a kernel that ignores the buffer's length writes past it, into the guard bytes)."""
    for name, case, out_len in geometries(pix):
        if name == "A/stride8":
            continue
        p, src, m, dst = build(case, pix, "opencv_fisheye", None, "Bilinear", out_len)
        runs = []
        for fill in (0xA5, 0x5A):
            out = np.full(out_len, fill, np.uint8)
            assert oracle_lib.undistort_image(src, out, p, pix, "opencv_fisheye", None, m) == 0
            runs.append(out)
        written = runs[0] == runs[1]                     # a byte the oracle leaves alone keeps its (different) fill
        bpp, _ = _bpp_align(pix)
        row = (out_len - 1) // p.output_stride * p.output_stride
        if name.endswith("ends-at-last-pixel"):
            assert written[out_len - bpp:].all(), name
        else:
            assert written[row + (CUT - 1) * bpp:row + CUT * bpp].all() and not written[row + CUT * bpp:].any(), name


def test_switches_leave_the_default_plan_alone(monkeypatch):
    """GF_DISABLE_LEAN off: the planner's choices are the ones it always made; on: general everywhere, two-pass kept."""
    from tests.test_abi import _plan
    set_switch(monkeypatch, None)
    base = dict(w=640, h=360)
    assert _plan(base) == 3 and _plan(dict(base, interp="EWA: Mitchell")) == 0x11
    monkeypatch.setenv("GF_DISABLE_LEAN", "1")
    assert _plan(base) == 0 and _plan(base, table_flags=1) == 0 and _plan(dict(base, lens="gopro", digital="gopro_warp")) == 0
    assert _plan(dict(base, interp="Lanczos4")) == 0x10 and _plan(dict(base, interp="EWA: Mitchell")) == 0x10
    assert _plan(dict(base, pix="R32f"), n_planes=4) == 0x10


# ---- the GPU matrix --------------------------------------------------------------------------------------------------------------
def render(case, pix, lens, digital, interp, tables, out_len, kinds):
    """Render one cell for each buffer kind in `kinds` ("host" / "device") on one context.  Returns (want, [(kind, got incl. guard,
    launches)], plan code).  A case with a mesh (cases.build's mesh / fpd keys) renders with it; DEVICE buffers keep the case's
    src_offset / dst_offset."""
    import torch
    p, src, m, dst = build(case, pix, lens, digital, interp, out_len)
    mesh = cases.build(dict(case, pix=pix, lens=lens, digital=digital, interp=interp))[3] if case.get("mesh") else None
    mesh_len = 0 if mesh is None else mesh.size
    want = dst[:out_len].copy()
    assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
    itm = g.FrameTransform(matrices=m, kernel_params=p, **({} if mesh is None else dict(mesh_data=mesh)))
    host = descs(case, p, src, dst, out_len)
    code = plan(p, pix, lens, digital, host, g.load_library().gf_table_flags_host(m.ctypes.data, m.shape[0]) if tables == "host" else 1, mesh_len)
    ctx = g.CudaWrapper.new(p, pix, lens, digital, host)
    tm = torch.from_numpy(m).cuda() if tables == "device" else None
    tmesh = torch.from_numpy(mesh).cuda() if tables == "device" and mesh is not None else None

    def dev(a, off):                    # a device copy of `a` that starts `off` bytes past an allocation's (256-byte aligned) start
        t = torch.empty(a.size + off, dtype=torch.uint8, device="cuda")
        t[off:].copy_(torch.from_numpy(a.copy()))
        return t[off:]
    outs = []
    try:
        for kind in kinds:
            if kind == "host":
                d = dst.copy(); bufs = descs(case, p, src, d, out_len)
            else:
                tsrc, d = dev(src, case.get("src_offset", 0)), dev(dst, case.get("dst_offset", 0))
                bufs = descs(case, p, tsrc, d, out_len)
            torch.cuda.synchronize()
            l0 = ctx.launch_count
            if tables == "host":
                ctx.undistort_image(bufs, itm)
            else:
                ctx.undistort_image_dev(bufs, p, tm.data_ptr(), m.shape[0], tmesh.data_ptr() if tmesh is not None else 0, mesh_len)
            ctx.synchronize()
            outs.append((kind, d if kind == "host" else d.cpu().numpy(), ctx.launch_count - l0))
    finally:
        ctx.close()
    return want, outs, code


def _first_bad(want, got, p_stride, bpp):
    idx = int(np.flatnonzero(want != got)[0])
    row, col = divmod(idx, p_stride)
    return "byte %d (row %d, pixel %d, byte %d of the pixel): want %d got %d" % (idx, row, col // bpp, col % bpp, want[idx], got[idx])


def run_matrix(request, monkeypatch, geometry_names, kinds, pairs=None, pixel_types=None, modes=None, extra=None, label=None):
    """Render every cell of pairs x pixel_types x modes in the named geometries with every buffer kind of `kinds`; reports the count,
    the time and every failing cell, fails with the first bad render, returns the set of cells rendered."""
    t0 = time.perf_counter()
    rendered, skipped, bad, bad_cells, renders = set(), set(), [], set(), 0
    pairs = pairs or library_pairs()
    for lens, digital in pairs:
        for pix in pixel_types or PIXEL_TYPES:
            bpp, _ = _bpp_align(pix)
            for name, case, out_len in geometries(pix):
                if name not in geometry_names:
                    continue
                case = dict(case, **(extra or {}))
                for mode, switch, interp, tables, code in modes or MODES:
                    set_switch(monkeypatch, switch)
                    cell = (lens, digital, pix, mode)
                    if interp.startswith("EWA") and (lens, digital, name[0]) in EWA_UNCOMPARABLE:
                        skipped.add(cell)
                        continue
                    want, outs, got_code = render(case, pix, lens, digital, interp, tables, out_len, kinds)
                    assert got_code == code, (cell, name, got_code, code)
                    for kind, got, launches in outs:
                        renders += 1
                        where = "%s %s %s" % (cell, name, kind)
                        assert launches == expected_launches(code, interp, lens, digital), (where, launches)
                        if not np.array_equal(got[out_len:], np.full(GUARD, 0xA5, np.uint8)):
                            bad.append("%s: wrote past the end of the output" % where)
                            bad_cells.add(cell)
                        elif not np.array_equal(got[:out_len], want):
                            stride = cases.build(dict(case, pix=pix, lens=lens, digital=digital))[0].output_stride
                            bad.append("%s: %d bytes differ, first at %s" % (where, int((got[:out_len] != want).sum()), _first_bad(want, got[:out_len], stride, bpp)))
                            bad_cells.add(cell)
                    rendered.add(cell)
    n_modes = len(modes or MODES)
    report(request, "%s: %d cells (%d pairs x %d pixel types x %d variants, %d EWA cells not comparable), %d renders, %d failing renders in %d cells, %.1f s" %
           (label or request.node.name, len(rendered), len(pairs), len(pixel_types or PIXEL_TYPES), n_modes, len(skipped), renders, len(bad), len(bad_cells),
            time.perf_counter() - t0))
    for c in sorted(bad_cells, key=str)[:64]:
        report(request, "  failing cell: %s %s %s %s" % c)
    assert not bad, "%d failing renders; first: %s" % (len(bad), bad[0])
    assert len(rendered) + len(skipped) == len(pairs) * len(pixel_types or PIXEL_TYPES) * n_modes
    return rendered


@pytest.mark.gpu
def test_matrix_identity_maps_odd_size(request, monkeypatch):
    """Geometry A: 75 x 43, identity output maps, a stride that is a multiple of 8 with the whole buffer, one that is not with
    buffers ending at the last pixel and part-way through the last row; HOST and DEVICE outputs, guard bytes untouched."""
    rendered = run_matrix(request, monkeypatch, ("A/stride8", "A/ends-at-last-pixel", "A/ends-mid-row"), ("host", "device"))
    assert len(rendered) == 21 * 13 * 9


@pytest.mark.gpu
def test_matrix_rects_and_short_output(request, monkeypatch):
    """Geometry B: source rect, output rect and size, fov 1.3, output buffers ending at the last (written) pixel and part-way through
    the last row; HOST and DEVICE outputs, guard bytes after the described length untouched."""
    rendered = run_matrix(request, monkeypatch, ("B/ends-at-last-pixel", "B/ends-mid-row"), ("host", "device"))
    assert len(rendered) == 21 * 13 * 9 - 13 * 2          # EWA_UNCOMPARABLE: one pair in both EWA variants


# ---- value-domain edges ----------------------------------------------------------------------------------------------------------
EDGE_PAIRS = [("opencv_fisheye", None), ("sony", "digital_stretch")]
EDGE_PIXEL_TYPES = ["R32f", "RGBAf", "RGBAf16", "Luma16", "RGBA16"]
RESAMPLERS = ("Bilinear", "Bicubic", "Lanczos4", "EWA: Mitchell")
EWA_FILTERS = ("EWA: RobidouxSharp", "EWA: Robidoux", "EWA: Mitchell", "EWA: Catmull-Rom")


def edge_modes():
    """Every variant of MODES with every resampler it can run: bilinear the four fused variants; bicubic, Lanczos4 and the four EWA
    filters the coordinate variants, EWA having no packed one."""
    out = [m for m in MODES if m[2] == "Bilinear"]
    for interp in RESAMPLERS[1:3] + EWA_FILTERS:
        for mode, switch, _, tables, code in MODES[4:7]:
            if interp.startswith("EWA") and mode == "packed-coords":
                continue
            out.append((mode + "/" + interp, switch, interp, tables, code))
    return out


# options only the general kernel has, once per resampler: pixel_value_limit below every format's maximum (it bites on 16-bit
# checkerboards and on the HDR / Inf float content) and background_mode 3 (feather)
GENERAL_OPTIONS = [("pixel_value_limit", dict(pixel_value_limit=1000.0)),
                   ("feather", dict(background_mode=3, background_margin=0.1, background_margin_feather=0.15, background=[0.25, 0.5, 0.75, 1.0]))]


@pytest.mark.gpu
def test_edge_values(request, monkeypatch):
    """HDR values, f16 values near 65504 (Lanczos overshoot to Inf on store), negatives, subnormals, +-0, +-Inf and NaNs with assorted
    payloads in R32f / RGBAf / RGBAf16, and 0 / 65535 checkerboards in Luma16 / RGBA16: every variant with every resampler, and the
    pixel_value_limit and feather options, byte-identical to the oracle (geometry A, fov 1.3)."""
    edge = dict(edge_values=True, fov=1.3)
    rendered = run_matrix(request, monkeypatch, ("A/stride8",), ("host",), pairs=EDGE_PAIRS, pixel_types=EDGE_PIXEL_TYPES,
                          modes=edge_modes(), extra=edge, label="test_edge_values, variants")
    assert len(rendered) == 2 * 5 * (4 + 3 + 3 + 4 * 2)
    for what, params in GENERAL_OPTIONS:
        modes = [(what + "/" + interp, None, interp, "host", 0 if interp == "Bilinear" else 0x10) for interp in RESAMPLERS]
        rendered = run_matrix(request, monkeypatch, ("A/stride8",), ("host",), pairs=EDGE_PAIRS, pixel_types=EDGE_PIXEL_TYPES,
                              modes=modes, extra=dict(edge, params=params), label="test_edge_values, " + what)
        assert len(rendered) == 2 * 5 * 4
