"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle, bit-exact.

Every test here needs a real H100 (`-m gpu`).  A missing GPU or a missing libgyroflow_cuda.so is a FAILURE,
never a skip: there is no fallback path to test instead.
"""
import os

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi, synth
from tests import cases, np_producer, oracle_lib

pytestmark = pytest.mark.gpu


def run_both(case, device_buffers=False):
    p, src, m, mesh, dst0, pix, lens, digital = cases.build(case)
    want = dst0.copy()
    rc = oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh)
    assert rc == 0, "oracle rc %d" % rc
    got = dst0.copy()
    bw, bh = case.get("in_size", (case["w"], case["h"]))
    obw, obh = case.get("out_size", (case.get("ow", case["w"]), case.get("oh", case["h"])))
    itm = g.FrameTransform(matrices=m, kernel_params=p, mesh_data=mesh if mesh is not None else np.zeros(0, np.float32))
    if not device_buffers:
        bufs = g.Buffers(g.BufferDescription((bw, bh, p.stride), src), g.BufferDescription((obw, obh, p.output_stride), got))
        w = g.CudaWrapper.new(p, pix, lens, digital, bufs)
        w.undistort_image(bufs, itm)
        # bilinear: one fused launch; other resamplers: coordinate pass(es) + sampling pass (EWA: pixel + two Jacobian probes);
        # a frame on the filtered pre-pass (packed fisheye kernel, rolling shutter on) adds the tail launch that renders the deferred pairs
        interp = case.get("interp", "Bilinear")
        base = 1 if interp == "Bilinear" else (4 if interp.startswith("EWA") else 2)
        assert w.launch_count in (base, base + 1), w.launch_count
        if w.launch_count == base + 1:
            assert lens == "opencv_fisheye" and digital is None and m.shape[0] > 1 and not interp.startswith("EWA") and not os.environ.get("GF_DISABLE_FILTER")
        w.close()
    else:
        import torch
        tsrc = torch.from_numpy(src).cuda()
        tdst = torch.from_numpy(got).cuda()
        bufs = g.Buffers(g.BufferDescription((bw, bh, p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                         g.BufferDescription((obw, obh, p.output_stride), tdst.data_ptr(), length=tdst.numel()))
        w = g.CudaWrapper.new(p, pix, lens, digital, bufs)
        side = torch.cuda.Stream()
        torch.cuda.synchronize()                     # uploads done before the side stream starts
        w.undistort_image(bufs, itm, stream=side.cuda_stream)
        side.synchronize()
        got = tdst.cpu().numpy()
        w.close()
    return want, got, pix


def assert_bit_exact(case, **kw):
    want, got, pix = run_both(case, **kw)
    n, mx = cases.compare(want, got, pix)
    assert n == 0, "%d mismatching bytes (max abs diff %s) for %r" % (n, mx, case)
    assert (want != 0xA5).any()     # the oracle really wrote something


def test_device_present():
    assert g.load_library().gf_cuda_device_count() > 0
    assert g.list_devices()[0].startswith("[CUDA] ")


# ---- BASELINE configs at reduced size (full size: test_full_size_*) --------------------------------------
def test_cfg1_fisheye_rs_off_identity():
    assert_bit_exact(dict(w=640, h=360, identity=True, rs=False))


def test_cfg2_fisheye_rolling_shutter():
    assert_bit_exact(dict(w=640, h=360))
    assert_bit_exact(dict(w=640, h=360, ts=2345.6))


def test_cfg3_luma16_superview_planes():
    assert_bit_exact(dict(w=960, h=540, pix="Luma16", digital="gopro_superview", fov=1.07))
    # 4:2:2 chroma plane: half-width buffer with source/output rect scaling (stabilization/mod.rs:230-231)
    assert_bit_exact(dict(w=960, h=540, pix="Luma16", digital="gopro_superview", fov=1.07, in_size=(480, 540), out_size=(480, 540)))


def test_cfg4_f32_sony_ibis_mesh():
    for pix in ("R32f", "RGBAf"):
        assert_bit_exact(dict(w=480, h=270, pix=pix, lens="sony", ibis=True, mesh=True))
    assert_bit_exact(dict(w=480, h=270, pix="R32f", lens="sony", ibis=True, mesh=True, fpd=True))


# ---- lens-model plugins ----------------------------------------------------------------------------------
@pytest.mark.parametrize("lens", ["opencv_fisheye", "opencv_standard", "poly3", "poly5", "ptlens", "insta360", "sony",
                                  "generic_polynomial", "gopro"])
def test_every_lens_model(lens):
    assert_bit_exact(dict(w=320, h=180, lens=lens))
    assert_bit_exact(dict(w=320, h=180, lens=lens, digital="gopro_warp" if lens == "gopro" else "digital_stretch"))
    # lens_correction_amount < 1 exercises undistort_point (Newton solvers, tanf)
    assert_bit_exact(dict(w=320, h=180, lens=lens, params=dict(lens_correction_amount=0.35)))


@pytest.mark.parametrize("digital", ["gopro_superview", "gopro6_superview", "gopro_hyperview", "digital_stretch"])
def test_fisheye_digital_lenses(digital):
    assert_bit_exact(dict(w=320, h=180, digital=digital))
    assert_bit_exact(dict(w=320, h=180, digital=digital, params=dict(lens_correction_amount=0.5)))


# ---- pixel formats ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("pix", sorted(abi.PIXEL_TYPES))
def test_every_pixel_format(pix):
    assert_bit_exact(dict(w=200, h=120, pix=pix))
    assert_bit_exact(dict(w=203, h=117, pix=pix, stride_pad=3))       # odd size, unaligned stride -> byte path


# ---- ragged / edge geometry ------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", [(4, 4), (5, 7), (33, 9), (31, 65), (257, 131), (1000, 4)])
def test_small_and_odd_sizes(w, h):
    assert_bit_exact(dict(w=w, h=h))
    assert_bit_exact(dict(w=w, h=h, identity=True, rs=False, stride_pad=1))


def test_output_size_differs_from_input():
    assert_bit_exact(dict(w=640, h=360, ow=480, oh=270))
    assert_bit_exact(dict(w=320, h=240, ow=640, oh=360, pix="Luma8"))


def test_rects():
    assert_bit_exact(dict(w=320, h=180, in_size=(400, 200), in_rect=(40, 10, 320, 180)))
    assert_bit_exact(dict(w=320, h=180, out_size=(400, 220), out_rect=(30, 20, 320, 180)))      # untouched border must survive
    assert_bit_exact(dict(w=320, h=180, pix="UV8", in_size=(160, 90), out_size=(160, 90)))      # NV12 chroma plane


# ---- per-frame features ----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [1, 2, 3])
def test_background_modes(mode):
    prm = dict(background_mode=mode, background=[0.1, 0.4, 0.7, 1.0])
    if mode == 3:
        prm.update(background_margin=0.2, background_margin_feather=0.1)
    assert_bit_exact(dict(w=320, h=180, fov=1.6, params=prm))


def test_background_colour_and_zoomed_out():
    assert_bit_exact(dict(w=320, h=180, fov=2.2, params=dict(background=[0.2, 0.4, 0.6, 1.0])))


def test_input_rotation_and_video_rotation():
    assert_bit_exact(dict(w=320, h=180, params=dict(input_rotation=90.0)))
    assert_bit_exact(dict(w=320, h=180, params=dict(input_rotation=-13.5, background_mode=2)))
    assert_bit_exact(dict(w=320, h=180, video_rotation=25.0))


def test_horizontal_rolling_shutter():
    assert_bit_exact(dict(w=320, h=180, horizontal_rs=True))


def test_light_refraction_and_r_limit():
    assert_bit_exact(dict(w=320, h=180, params=dict(light_refraction_coefficient=1.33)))
    assert_bit_exact(dict(w=320, h=180, params=dict(light_refraction_coefficient=1.33, lens_correction_amount=0.6)))
    assert_bit_exact(dict(w=320, h=180, fov=2.5, params=dict(r_limit=0.9)))


def test_fix_color_range_and_fill_background():
    assert_bit_exact(dict(w=320, h=180, pix="Luma8", flags=abi.FLAG_FIX_COLOR_RANGE))
    assert_bit_exact(dict(w=320, h=180, pix="UV8", flags=abi.FLAG_FIX_COLOR_RANGE, params=dict(plane_index=1)))
    assert_bit_exact(dict(w=320, h=180, flags=abi.FLAG_FILL_WITH_BACKGROUND, params=dict(background=[0.3, 0.6, 0.9, 1.0])))


def test_input_stretch_and_translation():
    assert_bit_exact(dict(w=320, h=180, params=dict(input_horizontal_stretch=1.3333, input_vertical_stretch=0.9, translation2d=[4.5, -3.25])))


def test_ibis_and_mesh_on_u8():
    assert_bit_exact(dict(w=320, h=180, ibis=True))
    assert_bit_exact(dict(w=320, h=180, mesh=True, fpd=True, flags=abi.FLAG_FRAMEBUFFER_INVERTED))


def test_mesh_spline_variants():
    """Unrolled 9-row spline (both extrapolation branches via a zoomed-out view), smaller grids through the general routine."""
    assert_bit_exact(dict(w=320, h=180, mesh=True, pix="RGBAf", lens="sony"))
    assert_bit_exact(dict(w=320, h=180, mesh=True, fov=1.8, lens="sony"))
    assert_bit_exact(dict(w=320, h=180, mesh=True, fpd=True, fov=0.7, pix="Luma16"))
    assert_bit_exact(dict(w=320, h=180, mesh=True, mesh_n=7, lens="sony"))
    assert_bit_exact(dict(w=320, h=180, mesh=True, mesh_n=5, fpd=True, ibis=True, lens="sony", pix="R32f"))


# ---- multi-plane frames (SURVEY f3): coordinates once, every plane sampled from the map -----------------------------------------
def _run_planes(case, n_planes, vary=None):
    """n planes with the case's geometry and different content / plane_index (/ background); returns [(want, got)] per plane."""
    import torch
    built = [cases.build(dict(case, frame=i)) for i in range(n_planes)]
    p0, _, m, mesh, dst0, pix, lens, digital = built[0]
    tm = torch.from_numpy(m).cuda()
    tmesh = torch.from_numpy(mesh).cuda() if mesh is not None else None
    params, bufs, keep, wants = [], [], [], []
    for i, (p, src, _, _, d0, _, _, _) in enumerate(built):
        p = p.copy(); p.plane_index = i
        if vary: vary(p, i)
        want = d0.copy()
        assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
        tsrc, tdst = torch.from_numpy(src).cuda(), torch.from_numpy(d0.copy()).cuda()
        bw, bh = case.get("in_size", (case["w"], case["h"]))
        obw, obh = case.get("out_size", (case.get("ow", case["w"]), case.get("oh", case["h"])))
        bufs.append(g.Buffers(g.BufferDescription((bw, bh, p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                              g.BufferDescription((obw, obh, p.output_stride), tdst.data_ptr(), length=tdst.numel())))
        params.append(p); keep.append((tsrc, tdst)); wants.append(want)
    w = g.CudaWrapper.new(params[0], pix, lens, digital, bufs[0])
    side = torch.cuda.Stream(); torch.cuda.synchronize()
    l0 = w.launch_count
    w.undistort_planes_dev(bufs, params, tm.data_ptr(), m.shape[0], tmesh.data_ptr() if tmesh is not None else 0, mesh.size if mesh is not None else 0,
                           stream=side.cuda_stream)
    side.synchronize()
    launches = w.launch_count - l0
    outs = [(wants[i], keep[i][1].cpu().numpy()) for i in range(n_planes)]
    w.close()
    return outs, launches, pix


def _assert_planes(case, n_planes, fused, vary=None):
    outs, launches, pix = _run_planes(case, n_planes, vary)
    interp = case.get("interp", "Bilinear")
    coord_passes = 3 if interp.startswith("EWA") else 1
    single = 1 if interp == "Bilinear" else coord_passes + 1
    want_l = coord_passes + n_planes if fused else n_planes * single
    assert launches in (want_l, want_l + 1, want_l + n_planes), launches          # + tail launch(es) of the filtered pre-pass (fisheye + rolling shutter)
    for i, (want, got) in enumerate(outs):
        n, mx = cases.compare(want, got, pix)
        assert n == 0, "plane %d: %d mismatching bytes (max abs diff %s) for %r" % (i, n, mx, case)


def test_fused_planes_gbrapf32_like():
    """Four R32f planes (GBRAPF32, cfg 4): sony lens + IBIS + mesh, one coordinate pass, four sampling passes."""
    _assert_planes(dict(w=320, h=180, pix="R32f", lens="sony", ibis=True, mesh=True), 4, fused=True)


def test_fused_planes_yuv_chroma_pair():
    """U and V of planar 16-bit YUV 4:2:2: half-width planes described by source / output rects (stabilization/mod.rs:209-231)."""
    case = dict(w=320, h=180, pix="Luma16", digital="gopro_superview", in_size=(160, 180), in_rect=(0, 0, 160, 180),
                out_size=(160, 180), out_rect=(0, 0, 160, 180))
    _assert_planes(case, 2, fused=True)


def test_fused_planes_options():
    fix = lambda p, i: setattr(p, "flags", p.flags | abi.FLAG_FIX_COLOR_RANGE)                    # is_y differs per plane (plane_index)
    _assert_planes(dict(w=320, h=180, pix="Luma8"), 3, fused=True, vary=fix)
    bgv = lambda p, i: p.background.__setitem__(slice(0, 4), [0.1 * (i + 1), 0.5, 0.25, 1.0])     # per-plane background colour
    _assert_planes(dict(w=320, h=180, pix="Luma16", fov=2.2), 3, fused=True, vary=bgv)
    _assert_planes(dict(w=320, h=180, pix="RGBA8", interp="Lanczos4"), 2, fused=True)
    _assert_planes(dict(w=320, h=180, pix="Luma8", params=dict(background_mode=3, background_margin=0.1, background_margin_feather=0.1), fov=1.6), 2, fused=True)
    _assert_planes(dict(w=320, h=180, pix="Luma8", flags=abi.FLAG_FILL_WITH_BACKGROUND, params=dict(background=[0.3, 0.3, 0.3, 1.0])), 2, fused=True)
    _assert_planes(dict(w=203, h=117, pix="UV8", stride_pad=2), 2, fused=True)
    _assert_planes(dict(w=200, h=120, pix="Luma8", interp="EWA: Mitchell"), 2, fused=True)         # three coordinate maps, shared
    # not fusable: planes whose parameters differ -> n ordinary calls, same results
    diff = lambda p, i: setattr(p, "lens_correction_amount", 1.0 if i == 0 else 0.5)
    _assert_planes(dict(w=320, h=180, pix="Luma8"), 2, fused=False, vary=diff)


def test_host_planes_entry_point():
    """gf_cuda_undistort_planes: the planes of a frame as HOST slices (what rendering/mod.rs:596-629 hands over) — staged, fused where the
    geometry is shared, copied back; bytes equal to per-plane oracle runs, untouched stride padding preserved."""
    for case, n in ((dict(w=320, h=180, pix="R32f", lens="sony", ibis=True, mesh=True), 4),
                    (dict(w=320, h=180, pix="Luma16", digital="gopro_superview", in_size=(160, 180), in_rect=(0, 0, 160, 180), out_size=(160, 180), out_rect=(0, 0, 160, 180)), 2),
                    (dict(w=203, h=117, pix="Luma8", stride_pad=5), 3)):
        built = [cases.build(dict(case, frame=i)) for i in range(n)]
        p0, _, m, mesh, dst0, pix, lens, digital = built[0]
        params, bufs, gots, wants = [], [], [], []
        bw, bh = case.get("in_size", (case["w"], case["h"])); obw, obh = case.get("out_size", (case["w"], case["h"]))
        for i, (p, src, _, _, d0, _, _, _) in enumerate(built):
            p = p.copy(); p.plane_index = i
            want = d0.copy()
            assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
            got = d0.copy()
            bufs.append(g.Buffers(g.BufferDescription((bw, bh, p.stride), src), g.BufferDescription((obw, obh, p.output_stride), got)))
            params.append(p); gots.append(got); wants.append(want)
        w = g.CudaWrapper.new(params[0], pix, lens, digital, bufs[0])
        w.undistort_planes(bufs, params, g.FrameTransform(matrices=m, kernel_params=params[0], mesh_data=mesh if mesh is not None else np.zeros(0, np.float32)))
        w.close()
        for i in range(n):
            assert np.array_equal(gots[i], wants[i]), (case, i)


# ---- higher-order resamplers (SURVEY f1): bicubic, Lanczos4 (the default render setting), EWA CubicBC ------------------
@pytest.mark.parametrize("interp", ["Bicubic", "Lanczos4"])
def test_bicubic_and_lanczos4(interp):
    assert_bit_exact(dict(w=640, h=360, interp=interp))
    assert_bit_exact(dict(w=320, h=180, interp=interp, pix="Luma16", lens="sony"))
    assert_bit_exact(dict(w=320, h=180, interp=interp, pix="RGBAf", lens="gopro", digital="gopro_warp"))
    assert_bit_exact(dict(w=203, h=117, interp=interp, pix="RGB8", stride_pad=3, fov=2.5))              # zoomed out: taps cross the source edge
    assert_bit_exact(dict(w=320, h=180, interp=interp, params=dict(background_mode=3, background_margin=0.1, background_margin_feather=0.1), fov=1.6))
    assert_bit_exact(dict(w=320, h=180, interp=interp, in_size=(400, 260), in_rect=(40, 30, 320, 180), out_size=(352, 200), out_rect=(16, 10, 320, 180)))
    assert_bit_exact(dict(w=320, h=180, interp=interp, pix="UV16", flags=abi.FLAG_FIX_COLOR_RANGE, params=dict(pixel_value_limit=60000.0)))


@pytest.mark.parametrize("pix", ["Luma8", "UV8", "RGBA8", "BGRA8", "Luma16", "UV16", "RGB8", "RGB16", "RGBA16", "AYUV16"])
@pytest.mark.parametrize("interp", ["Bicubic", "Lanczos4"])
def test_high_order_every_integer_format(interp, pix):
    """Row-window loader of the 16 / 64-tap samplers (RowWindow in warp_kernel.cuh: aligned 8-byte words + register re-alignment for formats
    of <= 4 bytes per pixel) against the oracle: 8-byte aligned strides (window path, every tap offset occurs), an odd width with a padded
    stride (the row's last aligned word is only partly valid), and strides that are not multiples of 8 (bounds-checked sampler instead)."""
    assert_bit_exact(dict(w=200, h=120, interp=interp, pix=pix))
    assert_bit_exact(dict(w=203, h=117, interp=interp, pix=pix, stride_pad=8 - (203 * abi.PIXEL_TYPES[pix][1] * np.dtype(abi.PIXEL_TYPES[pix][2]).itemsize) % 8, fov=1.3))
    assert_bit_exact(dict(w=202, h=90, interp=interp, pix=pix, stride_pad=2 if abi.PIXEL_TYPES[pix][2] == "u2" or pix == "UV8" else 1, rs=False))


@pytest.mark.parametrize("interp", ["EWA: RobidouxSharp", "EWA: Robidoux", "EWA: Mitchell", "EWA: Catmull-Rom"])
def test_ewa_cubic_bc(interp):
    assert_bit_exact(dict(w=320, h=180, interp=interp))
    assert_bit_exact(dict(w=200, h=120, interp=interp, pix="Luma16", lens="opencv_standard", rs=False))
    assert_bit_exact(dict(w=200, h=120, interp=interp, pix="RGBAf", fov=1.4, params=dict(background=[0.2, 0.4, 0.6, 1.0])))
    assert_bit_exact(dict(w=200, h=120, interp=interp, ow=100, oh=60))                                   # 2x minification: wide ellipses


def test_lanczos4_full_size_4k():
    assert_bit_exact(dict(w=3840, h=2160, interp="Lanczos4"))


# ---- buffer sources --------------------------------------------------------------------------------------
def test_device_buffers_cuda_buffer_source():
    assert_bit_exact(dict(w=640, h=360), device_buffers=True)
    assert_bit_exact(dict(w=203, h=117, pix="RGB8", stride_pad=3), device_buffers=True)


def test_host_register_in_place():
    """gf_cuda_host_register: an ordinary host array page-locked in place renders the same bytes; double registration is not an error."""
    p, src, m, mesh, dst0, pix, lens, digital = cases.build(dict(w=640, h=360))
    want = dst0.copy()
    assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
    got = dst0.copy()
    g.host_register(src); g.host_register(got); g.host_register(got)
    bufs = g.Buffers(g.BufferDescription((640, 360, p.stride), src), g.BufferDescription((640, 360, p.output_stride), got))
    w = g.CudaWrapper.new(p, pix, lens, digital, bufs)
    w.undistort_image(bufs, g.FrameTransform(matrices=m, kernel_params=p))
    w.close()
    g.host_unregister(src); g.host_unregister(got)
    assert np.array_equal(got, want)


# ---- full BASELINE sizes ---------------------------------------------------------------------------------
def test_full_size_cfg2_4k_rgba8():
    assert_bit_exact(dict(w=3840, h=2160))


def test_full_size_cfg3_8k_luma16():
    assert_bit_exact(dict(w=7680, h=4320, pix="Luma16", digital="gopro_superview", fov=1.05))


def test_full_size_cfg1_4k_rs_off_identity():
    """BASELINE config 1 at its real size: 3840x2160 RGBA8, opencv_fisheye, rolling shutter off, identity quaternion."""
    assert_bit_exact(dict(w=3840, h=2160, identity=True, rs=False))


def test_full_size_cfg4_4k_f32_sony_ibis_mesh():
    """BASELINE config 4 at its real size, both ways the reference renders f32: packed RGBAf in one call, and GBRAPF32 as four R32f
    planes through gf_cuda_undistort_planes_dev (one coordinate pass + four sampling passes, rendering/mod.rs:624-629)."""
    assert_bit_exact(dict(w=3840, h=2160, pix="RGBAf", lens="sony", ibis=True, mesh=True))
    _assert_planes(dict(w=3840, h=2160, pix="R32f", lens="sony", ibis=True, mesh=True), 4, fused=True)


def test_full_size_cfg3_8k_yuv422p16_with_adaptive_zoom():
    """BASELINE config 3 as the reference runs it: 7680x4320 YUV422P16LE = three Luma16 planes (7680x4320, 3840x4320, 3840x4320;
    rendering/mod.rs:596-610), opencv_fisheye + gopro_superview, rolling shutter on, and the per-frame fov taken from the adaptive-zoom
    companion: gf_cuda_find_fovs over the clip -> gf_zoom_dynamic_compute (window 4 s, envelope follower) -> fovs[frame]
    (zooming/mod.rs:35-70, frame_transform.rs:52-58)."""
    w, h = 7680, 4320
    p0 = synth.base_kernel_params(w, h, pixel_type="Luma16", digital_lens="gopro_superview")
    org, sm = cases.gyro()
    cp = g.ComputeParams(p0, org, sm)
    ts = np.arange(90) * (1000.0 / 60.0) + 500.0
    dg = g.DeviceGyro(cp)
    fov_min = dg.find_fovs("opencv_fisheye", "gopro_superview", ts)
    dg.close()
    fovs = g.zoom_dynamic(fov_min, 4.0, 60.0, 1)
    want_fovs = oracle_lib.zoom_dynamic(oracle_lib.find_fovs(cp, "opencv_fisheye", "gopro_superview", ts), 4.0, 60.0, 1)
    assert np.allclose(fovs, want_fovs, rtol=1e-6, atol=0)
    frame = 37
    fov = float(fovs[frame])
    assert 0.5 < fov < 1.5 and fovs.std() > 1e-4
    # luma plane, then the two half-width chroma planes (source / output rects, stabilization/mod.rs:209-231) fused into one coordinate pass
    assert_bit_exact(dict(w=w, h=h, pix="Luma16", digital="gopro_superview", fov=fov, ts=float(ts[frame])))
    chroma = dict(w=w, h=h, pix="Luma16", digital="gopro_superview", fov=fov, ts=float(ts[frame]),
                  in_size=(w // 2, h), in_rect=(0, 0, w // 2, h), out_size=(w // 2, h), out_rect=(0, 0, w // 2, h))
    _assert_planes(chroma, 2, fused=True)


# ---- size-independent properties at full size ------------------------------------------------------------
def test_property_frame_sharding_is_order_independent():
    """Frames are independent units: warping frames in any order / on a reused context gives identical bytes."""
    case = dict(w=1920, h=1080)
    p, src, m, mesh, dst0, pix, lens, digital = cases.build(case)
    bufs = lambda d: g.Buffers(g.BufferDescription((1920, 1080, p.stride), src), g.BufferDescription((1920, 1080, p.output_stride), d))
    w = g.CudaWrapper.new(p, pix, lens, digital, bufs(dst0))
    org, sm = cases.gyro()
    outs = {}
    for ts in (500.0, 1500.0, 500.0, 2500.0, 1500.0):
        mm = np_producer.frame_matrices(p, org, sm, ts)
        d = dst0.copy()
        w.undistort_image(bufs(d), g.FrameTransform(matrices=mm, kernel_params=p))
        if ts in outs:
            assert np.array_equal(outs[ts], d)
        outs[ts] = d
    assert not np.array_equal(outs[500.0], outs[1500.0])
    w.close()


# ---- error behaviour (mirrors GyroflowCoreError) ---------------------------------------------------------
def test_errors():
    p, src, m, mesh, dst, pix, lens, digital = cases.build(dict(w=64, h=36))
    bufs = g.Buffers(g.BufferDescription((64, 36, p.stride), src), g.BufferDescription((64, 36, p.output_stride), dst))
    with pytest.raises(g.GyroflowCoreError) as e:
        g.CudaWrapper.new(p, pix, "poly3", "gopro_superview", bufs)          # pair the reference never builds
    assert e.value.kind == "UnsupportedCombo"
    small = g.Buffers(g.BufferDescription((64, 3, p.stride), src), g.BufferDescription((64, 36, p.output_stride), dst))
    with pytest.raises(g.GyroflowCoreError) as e:
        g.CudaWrapper.new(p, pix, lens, digital, small)
    assert e.value.kind == "SizeTooSmall"
    w = g.CudaWrapper.new(p, pix, lens, digital, bufs)
    p2 = p.copy(); p2.width = 65
    with pytest.raises(g.GyroflowCoreError) as e:
        w.undistort_image(bufs, g.FrameTransform(matrices=m, kernel_params=p2))
    assert e.value.kind == "SizeMismatch"
    p3 = p.copy(); p3.source_rect[:] = [0, 0, 64, 400]
    with pytest.raises(g.GyroflowCoreError) as e:
        w.undistort_image(bufs, g.FrameTransform(matrices=m, kernel_params=p3))
    assert e.value.kind == "BufferTooSmall"
    with pytest.raises(g.GyroflowCoreError) as e:
        w.undistort_image(bufs, g.FrameTransform(matrices=m[:10], kernel_params=p))
    assert e.value.kind == "BufferTooSmall"
    w.close()


# ---- packed f32x2 primitives (device self-test) and kernel-variant agreement --------------------------------
def test_packed_primitives_selftest():
    """div / sqrt / atanf / uniform-divisor division on register pairs == the scalar IEEE operations, 2^28 operand sets."""
    import ctypes as C
    lib = g.load_library()
    out = (C.c_ulonglong * 4)()
    assert lib.gf_cuda_selftest(0, 1 << 28, 12345, out) == 0
    assert list(out) == [0, 0, 0, 0], list(out)


def test_filtered_prepass_certificate_on_device():
    """The filtered rolling-shutter pre-pass (Lens2<opencv_fisheye>::approx_v): on the real MUFU units, over 400 random lenses / mid-row
    matrices / frame sizes and every 3rd pixel, the approximate v never differs from the reference's float result by more than the
    proven bound rho |tv - c| + 2^-22 |tv| (0 violations), stays well inside it, and leaves only a few percent of the pixels uncertain."""
    import ctypes as C
    out = (C.c_ulonglong * 4)()
    assert g.load_library().gf_cuda_selftest_filter(0, 2024, 400, 3, out) == 0
    n, viol, unc, worst = [int(v) for v in out]
    assert n > 2e8, n
    assert viol == 0, (viol, worst)
    assert worst <= 500000, worst                  # max |diff| / bound <= 0.5: a factor two of margin on top of the analysis
    assert unc / n < 0.05, unc / n


def test_filtered_prepass_queue_overflow_and_extremes(monkeypatch):
    """Frames where the certificate fails for MANY pairs — strong roll (the row boundaries run diagonally through every warp), a lens at
    its conditioning cap, a view zoomed out past the cap, translation — still match the oracle: deferred pairs go through the tail
    launch.  None of these frames defers more pairs than the queue holds (1920 x 1080 has fewer pairs in all); the full queue's inline
    fallback and the tail's grid-stride loop are tested in tests/test_filter_queue.py, on frames proven to reach them."""
    for c in (dict(w=1920, h=1080, video_rotation=33.0), dict(w=1920, h=1080, fov=3.5, ts=1234.0), dict(w=1280, h=720, params=dict(k=[0.18, -0.06, 0.02, -0.004] + [0.0] * 8)),
              dict(w=1280, h=720, params=dict(k=[-0.21, 0.0, 0.0, 0.0] + [0.0] * 8), fov=1.7), dict(w=1280, h=720, params=dict(translation2d=[13.5, -7.25]), readout=33.0),
              dict(w=3840, h=2160, ts=3456.7, pix="Luma8"), dict(w=2048, h=1152, ow=1024, oh=576), dict(w=640, h=360, out_size=(700, 400), out_rect=(30, 20, 640, 360))):
        assert_bit_exact(c)
        assert_bit_exact(c, device_buffers=True)


def test_packed_sequences_exhaustive_on_device():
    """Every input of the packed atanf ([2^-28, 2^24): 4.4e8 floats) and of the packed square root ([2^-56, 2^48)) against the scalar
    functions, on the device (a few seconds; round 2 runs it unconditionally)."""
    import ctypes as C
    out = (C.c_ulonglong * 2)()
    assert g.load_library().gf_cuda_selftest_exhaustive(0, out) == 0
    assert list(out) == [0, 0], list(out)


def test_many_frames_and_rotations():
    """Many frames, strong shake, in-plane rotation, zoomed-out views with invalid (w <= 0) regions, odd sizes."""
    org, sm = cases.gyro()
    for i in range(12):
        assert_bit_exact(dict(w=1280, h=720, ts=137.0 + 311.7 * i))
    for rot in (3.0, 17.0, 45.0, 90.0, 179.0):
        assert_bit_exact(dict(w=1280, h=720, video_rotation=rot, ts=777.0))
    for fov in (0.4, 1.0, 3.0, 8.0):
        assert_bit_exact(dict(w=1031, h=577, fov=fov, ts=1999.0, readout=33.0))
    assert_bit_exact(dict(w=1280, h=720, readout=-20.0))
    assert_bit_exact(dict(w=70, h=41))
    assert_bit_exact(dict(w=1280, h=720, pix="Luma8"))
    assert_bit_exact(dict(w=1280, h=720, pix="RGBAf"))


def _wild(kind):
    def hook(m):
        n = m.shape[0]
        if kind == "nan_row":    m[n // 3, :9] = np.nan
        if kind == "inf":        m[n // 2, 2] = np.inf; m[(n // 2 + 1) % n, 8] = -np.inf
        if kind == "huge":       m[n // 4:n // 4 + 5, :9] *= np.float32(1e30)
        if kind == "tiny":       m[n // 4:n // 4 + 5, :9] *= np.float32(1e-30)
        if kind == "denormal":   m[n // 5, :9] *= np.float32(1e-38); m[(n // 5 + 1) % n, 6:9] = np.float32(1e-44)
        if kind == "zero_rows":  m[::7, :9] = 0.0
        if kind == "zero_w":     m[n // 2:n // 2 + 9, 6:9] = 0.0
        if kind == "negzero":    m[::5, 0:2] = -0.0
        if kind == "on_axis":    m[:, 0:2] = 0.0; m[:, 3:5] = 0.0; m[:, 2] = 0.0; m[:, 5] = 0.0       # x = y = 0 everywhere: r == 0 branch
        if kind == "ibis_some":  m[n // 2:, 9] = 2.5; m[n // 2:, 11] = 0.01
        if kind == "ibis_negzero": m[:, 9:14] = -0.0                                                 # -0.0 != 0.0 is false: not IBIS
        return m
    return hook


@pytest.mark.parametrize("kind", ["nan_row", "inf", "huge", "tiny", "denormal", "zero_rows", "zero_w", "negzero", "on_axis", "ibis_some", "ibis_negzero"])
def test_packed_kernel_cold_path_on_unusual_tables(kind):
    """Tables the packed kernel's fast sequences do not cover (non-finite / extreme entries, r == 0, IBIS rows under a fisheye
    lens) must take the exact scalar code and still match the CPU path byte for byte."""
    for rs in (True, False):
        assert_bit_exact(dict(w=640, h=360, rs=rs, matrix_hook=_wild(kind)))


@pytest.mark.parametrize("lens", ["sony", "opencv_standard", "poly3", "poly5", "ptlens", "generic_polynomial", "insta360"])
def test_packed_kernel_other_lens_models(lens):
    """The packed kernel also carries these lens models: ordinary frames, its cold path, all 8/16-bit/f32 layouts."""
    for pix in ("RGBA8", "Luma8", "UV16", "RGBAf", "RGB8"):
        assert_bit_exact(dict(w=640, h=360, lens=lens, pix=pix))
    assert_bit_exact(dict(w=1280, h=720, lens=lens, ts=2222.0, readout=33.0))
    assert_bit_exact(dict(w=640, h=360, lens=lens, rs=False))
    assert_bit_exact(dict(w=640, h=360, lens=lens, fov=3.0))                                   # invalid (w <= 0) regions -> cold path
    for kind in ("nan_row", "huge", "zero_w", "on_axis", "ibis_some"):
        assert_bit_exact(dict(w=320, h=180, lens=lens, matrix_hook=_wild(kind)))
    assert_bit_exact(dict(w=640, h=360, lens=lens, digital="digital_stretch"))                  # packed digital_stretch pair
    assert_bit_exact(dict(w=320, h=180, lens=lens, digital="digital_stretch", pix="Luma16", matrix_hook=_wild("zero_w")))
    if lens == "opencv_standard":      # denominators of the rational term crossing zero / huge coefficients
        assert_bit_exact(dict(w=640, h=360, lens=lens, fov=2.0, params=dict(k=[0.1, 0.01, 0.001, 0.001, 0.0, -3.0, 0.5, 0.0, 0.0, 0.0, 0.0, 0.0])))
        assert_bit_exact(dict(w=640, h=360, lens=lens, params=dict(k=[1e20, 0.0, 0.0, 0.0, 0.0, 1e20, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0])))


def test_packed_kernel_gopro_pair():
    """The packed forms of `gopro` (Newton POLY inversion with per-lane stop masks) and of its `gopro_warp` digital lens (12-step fixed
    point + off-frame sentinel): ordinary frames, every pixel layout family, rays past the 89-degree continuation, wild tables, odd k."""
    for digital in (None, "gopro_warp"):
        for pix in ("RGBA8", "Luma8", "UV16", "RGBAf", "RGB8"):
            assert_bit_exact(dict(w=640, h=360, lens="gopro", digital=digital, pix=pix))
        assert_bit_exact(dict(w=1280, h=720, lens="gopro", digital=digital, ts=2222.0, readout=33.0))
        assert_bit_exact(dict(w=640, h=360, lens="gopro", digital=digital, rs=False))
        assert_bit_exact(dict(w=640, h=360, lens="gopro", digital=digital, fov=3.0))                 # invalid (w <= 0) regions, rays past 89 degrees, off-frame sentinel
        assert_bit_exact(dict(w=640, h=360, lens="gopro", digital=digital, fov=0.5))
        for kind in ("nan_row", "huge", "zero_w", "on_axis", "ibis_some"):
            assert_bit_exact(dict(w=320, h=180, lens="gopro", digital=digital, matrix_hook=_wild(kind)))
    assert_bit_exact(dict(w=640, h=360, lens="gopro", params=dict(k=[0.0, 1.15, 0.3, -0.5, 0.9, 0.0, 0.0] + [0.0] * 5)))     # a POLY whose derivative changes sign in range
    assert_bit_exact(dict(w=640, h=360, lens="gopro", params=dict(k=[0.01, -1.15, 0.01, 0.12, -0.03, 0.02, 0.005] + [0.0] * 5)))
    assert_bit_exact(dict(w=640, h=360, lens="gopro", params=dict(k=[0.0, 1e-30, 0.0, 0.0, 0.0, 0.0, 0.0] + [0.0] * 5)))
    assert_bit_exact(dict(w=640, h=360, lens="gopro", digital="gopro_warp", params=dict(digital_lens_params=[1.55, -3.0, 9.0, -20.0, 30.0, -25.0, 9.0, 0.2, 1.0, 0.3, -0.5, -0.3, 0.9, 0.3, 1.5556, 0.0])))


def test_packed_kernel_unusual_params():
    assert_bit_exact(dict(w=640, h=360, params=dict(pixel_value_limit=200.0)))
    assert_bit_exact(dict(w=640, h=360, params=dict(k=[1e30, -1e30, 0.0, 0.0] + [0.0] * 8)))
    assert_bit_exact(dict(w=640, h=360, params=dict(k=[float("nan"), 0.1, 0.0, 0.0] + [0.0] * 8)))
    assert_bit_exact(dict(w=640, h=360, params=dict(k=[-0.3, 0.0, 0.0, 0.0] + [0.0] * 8)))         # theta_d crosses zero
    assert_bit_exact(dict(w=640, h=360, params=dict(translation2d=[1e6, -3.25])))
    assert_bit_exact(dict(w=640, h=360, params=dict(f=[1e-30, 1e30])))
    assert_bit_exact(dict(w=640, h=360, params=dict(c=[0.0, 0.0])))
    assert_bit_exact(dict(w=640, h=360, in_size=(640, 362), in_rect=(0, 1, 640, 1)))                  # 1-row source rect: no interior


def test_device_tables_validated_and_not():
    """gf_cuda_undistort_image_dev on device tables: without a verdict word (guarded path), with a word written by
    gf_cuda_scan_tables_dev (trusted path when 0) — both == oracle; the scan reports wild entries / IBIS rows and those tables still
    render exactly.  A table REWRITTEN IN PLACE is rendered correctly as long as its word is rewritten too (no pointer cache)."""
    import torch
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    for hook, verdict in ((None, 0), (_wild("huge"), 1), (_wild("ibis_some"), 2), (_wild("nan_row"), 1)):
        case = dict(w=1280, h=720)
        if hook: case["matrix_hook"] = hook
        p, src, m, mesh, dst0, pix, lens, digital = cases.build(case)
        want = dst0.copy()
        assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
        tsrc = torch.from_numpy(src).cuda(); tm = torch.from_numpy(m).cuda()
        outs = []
        for use_flags in (False, True):
            tdst = torch.from_numpy(dst0.copy()).cuda()
            bufs = g.Buffers(g.BufferDescription((1280, 720, p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                             g.BufferDescription((1280, 720, p.output_stride), tdst.data_ptr(), length=tdst.numel()))
            w = g.CudaWrapper.new(p, pix, lens, digital, bufs)
            torch.cuda.synchronize()
            side = torch.cuda.Stream()
            if use_flags:
                assert w.validate_tables_dev(tm.data_ptr(), m.shape[0]) == verdict          # synchronous query
                flags.fill_(-1); torch.cuda.synchronize()
                g.scan_tables_dev(tm.data_ptr(), m.shape[0], flags.data_ptr(), stream=side.cuda_stream)   # asynchronous, same stream as the warp
            w.undistort_image_dev(bufs, p, tm.data_ptr(), m.shape[0], stream=side.cuda_stream, table_flags_dev=flags.data_ptr() if use_flags else 0)
            side.synchronize()
            if use_flags: assert int(flags.item()) == verdict
            outs.append(tdst.cpu().numpy()); w.close()
        assert np.array_equal(outs[0], want) and np.array_equal(outs[1], want)
    # in-place rewrite: tame table scanned (word = 0), then IBIS rows written into the SAME allocation and re-scanned
    p, src, m, mesh, dst0, pix, lens, digital = cases.build(dict(w=640, h=360))
    m2 = _wild("ibis_some")(m.copy())
    tsrc = torch.from_numpy(src).cuda(); tm = torch.from_numpy(m).cuda()
    tdst = torch.from_numpy(dst0.copy()).cuda()
    bufs = g.Buffers(g.BufferDescription((640, 360, p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                     g.BufferDescription((640, 360, p.output_stride), tdst.data_ptr(), length=tdst.numel()))
    w = g.CudaWrapper.new(p, pix, lens, digital, bufs)
    side = torch.cuda.Stream(); torch.cuda.synchronize()
    for table in (m, m2, m):
        with torch.cuda.stream(side):
            tm.copy_(torch.from_numpy(table).cuda(), non_blocking=True)
        g.scan_tables_dev(tm.data_ptr(), table.shape[0], flags.data_ptr(), stream=side.cuda_stream)
        w.undistort_image_dev(bufs, p, tm.data_ptr(), table.shape[0], stream=side.cuda_stream, table_flags_dev=flags.data_ptr())
        side.synchronize()
        want = dst0.copy()
        assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, table, mesh) == 0
        assert np.array_equal(tdst.cpu().numpy(), want)
    w.close()


def test_kernel_variants_agree(monkeypatch):
    """The packed two-pixel kernel, the lean scalar kernel and the general kernel produce identical bytes."""
    case = dict(w=1280, h=720)
    want, got_x2, pix = run_both(case)
    assert cases.compare(want, got_x2, pix)[0] == 0
    monkeypatch.setenv("GF_DISABLE_FILTER", "1")                 # packed kernel with the exact pre-pass for every pair
    _, got_nofilter, _ = run_both(case)
    assert np.array_equal(got_x2, got_nofilter)
    monkeypatch.delenv("GF_DISABLE_FILTER")
    monkeypatch.setenv("GF_DISABLE_X2", "1")
    _, got_lean, _ = run_both(case)
    assert np.array_equal(got_x2, got_lean)
    monkeypatch.delenv("GF_DISABLE_X2")
    monkeypatch.setenv("GF_DISABLE_LEAN", "1")                   # the general kernel on the same plain frame
    _, got_gen, _ = run_both(case)
    assert np.array_equal(got_x2, got_gen)


def test_concurrent_contexts_from_host_threads():
    """process_pixels holds only a read lock (lib.rs:931): several host threads drive their own wrappers at the same time.
    Four threads, each with its own context / frame size / lens, 16 host-buffer frames each, all bit-exact."""
    import threading
    specs = [dict(w=640, h=360), dict(w=512, h=288, lens="sony", pix="Luma16"), dict(w=400, h=300, digital="gopro_superview", pix="UV8"),
             dict(w=320, h=180, pix="RGBAf", interp="Lanczos4")]
    errors = []

    def worker(spec):
        try:
            p, src, m0, mesh, dst0, pix, lens, digital = cases.build(spec)
            bufs_proto = (spec["w"], spec["h"])
            got = dst0.copy()
            bufs = g.Buffers(g.BufferDescription((bufs_proto[0], bufs_proto[1], p.stride), src), g.BufferDescription((bufs_proto[0], bufs_proto[1], p.output_stride), got))
            w = g.CudaWrapper.new(p, pix, lens, digital, bufs)
            for i in range(16):
                pi, _, mi, _, _, _, _, _ = cases.build(dict(spec, ts=200.0 + 97.0 * i))
                want = dst0.copy()
                assert oracle_lib.undistort_image(src, want, pi, pix, lens, digital, mi, mesh) == 0
                got[:] = dst0
                w.undistort_image(bufs, g.FrameTransform(matrices=mi, kernel_params=pi, mesh_data=np.zeros(0, np.float32)))
                n, mx = cases.compare(want, got, pix)
                if n:
                    errors.append((spec, i, n, mx)); break
            w.close()
        except Exception as e:       # noqa: BLE001 - reported below
            errors.append((spec, repr(e)))

    threads = [threading.Thread(target=worker, args=(s,)) for s in specs]
    for t in threads: t.start()
    for t in threads: t.join()
    assert not errors, errors


# ---- randomized sweep ------------------------------------------------------------------------------------------------------
_PAIRS = [("opencv_fisheye", d) for d in (None, "gopro_superview", "gopro6_superview", "gopro_hyperview", "digital_stretch")] + \
         [("gopro", None), ("gopro", "gopro_warp")] + \
         [(l, d) for l in ("opencv_standard", "poly3", "poly5", "ptlens", "insta360", "sony", "generic_polynomial") for d in (None, "digital_stretch")]


def _random_case(rng):
    lens, digital = _PAIRS[rng.integers(len(_PAIRS))]
    pix = sorted(abi.PIXEL_TYPES)[rng.integers(len(abi.PIXEL_TYPES))]
    w, h = int(rng.integers(8, 200)), int(rng.integers(8, 120))
    c = dict(w=w, h=h, lens=lens, digital=digital, pix=pix, ts=float(rng.uniform(100, 3500)), fov=float(rng.choice([0.6, 1.0, 1.0, 1.5, 2.5])),
             rs=bool(rng.integers(4) != 0), readout=float(rng.choice([16.0, 33.0, -12.0])), stride_pad=int(rng.choice([0, 0, 1, 3, 64])),
             interp=str(rng.choice(["Bilinear", "Bilinear", "Bicubic", "Lanczos4"])))
    params = {}
    r = rng.integers(10)
    if r == 0: params["background_mode"] = int(rng.integers(1, 4)); params["background_margin"] = 0.1; params["background_margin_feather"] = 0.05
    if r == 1: params["input_rotation"] = float(rng.choice([90.0, 180.0, 270.0, 33.0]))
    if r == 2: params["light_refraction_coefficient"] = 1.33
    if r == 3: params["lens_correction_amount"] = float(rng.uniform(0.0, 0.9))
    if r == 4: params["translation2d"] = [float(rng.uniform(-20, 20)), float(rng.uniform(-20, 20))]
    if r == 5: params["r_limit"] = float(rng.uniform(0.5, 2.0))
    if r == 6: params["input_horizontal_stretch"] = 1.1; params["input_vertical_stretch"] = 0.95
    if r == 7: params["background"] = [float(x) for x in rng.uniform(0, 1, 4)]
    if rng.integers(6) == 0: c["horizontal_rs"] = True
    if rng.integers(8) == 0: c["ibis"] = True
    if rng.integers(8) == 0: c["mesh"] = True; c["fpd"] = bool(rng.integers(2))
    if rng.integers(8) == 0: c["flags"] = int(rng.choice([abi.FLAG_FIX_COLOR_RANGE, abi.FLAG_FILL_WITH_BACKGROUND, abi.FLAG_FRAMEBUFFER_INVERTED]))
    if rng.integers(6) == 0:
        mx, my = int(rng.integers(0, 9)), int(rng.integers(0, 9))
        c["in_size"] = (w + 2 * mx, h + 2 * my); c["in_rect"] = (mx, my, w, h)
        c["out_size"] = (w + mx, h + my); c["out_rect"] = (mx // 2, my // 2, w, h)
    if params: c["params"] = params
    return c


@pytest.mark.parametrize("seed", range(4))
def test_randomized_fisheye_filter_sweep(seed):
    """The filtered pre-pass under random conditions: 30 frames per seed of the opencv_fisheye model with random coefficients (both signs, weak to
    beyond the conditioning cap), focal lengths, principal points, roll / readout times, zoom, translations, sizes and 8-bit layouts — every
    frame byte-identical to the CPU oracle (pairs the certificate cannot decide go through the tail launch or, past the cap, everything does)."""
    rng = np.random.default_rng(7000 + seed)
    for _ in range(30):
        w, h = int(rng.integers(64, 420)), int(rng.integers(48, 260))
        scale = float(rng.choice([0.02, 0.2, 1.0, 3.0]))
        k = [float(rng.normal(0, 0.08) * scale), float(rng.normal(0, 0.03) * scale), float(rng.normal(0, 0.01) * scale), float(rng.normal(0, 0.004) * scale)] + [0.0] * 8
        f = float(rng.uniform(0.25, 1.4) * w)
        params = dict(k=k, f=[f, f * float(rng.uniform(0.97, 1.03))], c=[w / 2 + float(rng.uniform(-20, 20)), h / 2 + float(rng.uniform(-20, 20))])
        if rng.integers(3) == 0: params["translation2d"] = [float(rng.uniform(-15, 15)), float(rng.uniform(-15, 15))]
        c = dict(w=w, h=h, pix=str(rng.choice(["RGBA8", "Luma8", "UV8", "RGB8", "Luma16"])), ts=float(rng.uniform(100, 3600)), fov=float(rng.choice([0.7, 1.0, 1.0, 1.3, 2.2])),
                 readout=float(rng.choice([8.0, 16.0, 33.0, -16.0])), video_rotation=float(rng.choice([0.0, 0.0, 2.0, 11.0, 45.0, 90.0])), params=params,
                 interp=str(rng.choice(["Bilinear", "Bilinear", "Bilinear", "Lanczos4"])))
        if c["pix"] == "RGB8": c["stride_pad"] = int(rng.choice([0, 1]))
        assert_bit_exact(c)


@pytest.mark.parametrize("seed", range(6))
def test_randomized_sweep(seed):
    """40 random combinations per seed of lens / digital lens / pixel format / resampler / size / stride / rects / per-frame options."""
    rng = np.random.default_rng(1000 + seed)
    for _ in range(40):
        assert_bit_exact(_random_case(rng))
