"""How the entry points behind the gyro object (point path, ST maps, adaptive zoom, matrix producer) report a refused argument: the
same code as always, and a gf_cuda_last_error(NULL) that names the entry point instead of whatever failed earlier on the thread.
Every call here is refused before any CUDA call, so none needs a GPU."""
import ctypes as C

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi, synth
from tests import cases

GF_ERR_BAD_PARAMS, GF_ERR_BUFFER_TOO_SMALL = -1, -7
FISHEYE = abi.LENS["opencv_fisheye"]

# each entry point with a NULL handle or argument where it checks one
NULL_CALLS = {
    "gf_cuda_find_fovs": lambda lib: lib.gf_cuda_find_fovs(None, None, FISHEYE, 0, None, 1, 2.0, None, None),
    "gf_cuda_undistort_points": lambda lib: lib.gf_cuda_undistort_points(None, None, FISHEYE, 0, 0.0, 0, 0, 1.0, None, 1, None, None),
    "gf_cuda_stmap_distort_dev": lambda lib: lib.gf_cuda_stmap_distort_dev(None, None, FISHEYE, 0, 0.0, 0, None, None),
    "gf_cuda_stmap_sizes": lambda lib: lib.gf_cuda_stmap_sizes(None, None, FISHEYE, 0, 1, None, None, 1, None, None, None),
    "gf_cuda_generate_stmap": lambda lib: lib.gf_cuda_generate_stmap(None, None, FISHEYE, 0, 1, 0, 0.0, None, None, None, 0, None, 0, None),
    "gf_cuda_generate_stmaps_dev": lambda lib: lib.gf_cuda_generate_stmaps_dev(None, None, FISHEYE, 0, 1, None, None, 1, None, None, None, None,
                                                                               0, 0, None),
    "gf_zoom_dynamic_compute": lambda lib: lib.gf_zoom_dynamic_compute(None, 1, 1.0, 30.0, 0, None),
    "gf_zoom_fovs": lambda lib: lib.gf_zoom_fovs(None, None, None, 1, None, None),
    "gf_cuda_calculate_fovs": lambda lib: lib.gf_cuda_calculate_fovs(None, None, None, FISHEYE, 0, None, 1, None, None, None),
    "gf_frame_transform_at_timestamp": lambda lib: lib.gf_frame_transform_at_timestamp(None, 0.0, 0, None, None, 0, None, None, None),
    "gf_cuda_gyro_upload": lambda lib: lib.gf_cuda_gyro_upload(None, 0, None),
    "gf_cuda_frame_transform_dev_flagged": lambda lib: lib.gf_cuda_frame_transform_dev_flagged(None, None, 0.0, 0, None, None, 0, None, None,
                                                                                               None, None, None),
    "gf_get_frame_transform_at": lambda lib: lib.gf_get_frame_transform_at(None, None, None, None, None, 0, 0.0, 0, 1.0, None),
}


def stale_message(lib):
    """Leave another failure's message on the thread: gf_cuda_create without a handle to write."""
    assert lib.gf_cuda_create(None, 0, None, 0, 0, 0, None, None, 0) == GF_ERR_BAD_PARAMS
    msg = lib.gf_cuda_last_error(None).decode()
    assert msg and not msg.startswith("gf_")
    return msg


def reported(lib, entry):
    msg = lib.gf_cuda_last_error(None).decode()
    assert msg.startswith(entry + ": "), msg
    return msg


@pytest.mark.parametrize("entry", sorted(NULL_CALLS))
def test_null_argument_names_the_entry_point(entry):
    lib = g.load_library()
    stale_message(lib)
    assert NULL_CALLS[entry](lib) == GF_ERR_BAD_PARAMS
    assert "null argument" in reported(lib, entry)


def test_short_matrix_buffer_names_the_entry_point():
    """The host producer with room for fewer rows than a rolling-shutter frame has: GF_ERR_BUFFER_TOO_SMALL, and the reason."""
    lib = g.load_library()
    cp = g.ComputeParams(synth.base_kernel_params(64, 36), *cases.gyro())
    m = np.zeros((1, 14), np.float32)
    rows = C.c_size_t()
    stale_message(lib)
    assert lib.gf_frame_transform_at_timestamp(C.byref(cp.c), 100.0, 0, None, m.ctypes.data, 1, C.byref(rows), None, None) == GF_ERR_BUFFER_TOO_SMALL
    assert rows.value == 36
    assert "max_rows" in reported(lib, "gf_frame_transform_at_timestamp")


def test_unknown_pixel_type_names_the_entry_point():
    lib = g.load_library()
    p = synth.base_kernel_params(64, 36)
    cp = g.ComputeParams(p, *cases.gyro())
    st = g.stab_config(p, "RGBA8")
    st.pixel_type = 99
    d = abi.BufferDesc()
    d.width, d.height, d.stride = 64, 36, p.stride
    kp = abi.KernelParams()
    stale_message(lib)
    assert lib.gf_get_frame_transform_at(C.byref(st), C.byref(cp.c), C.byref(d), C.byref(d), None, 0, 0.0, 0, 1.0, C.byref(kp)) == GF_ERR_BAD_PARAMS
    assert "pixel type" in reported(lib, "gf_get_frame_transform_at")


def test_zoom_window_too_long_raises_with_the_reason():
    """A static window of 3e8 frames is refused instead of allocated; the Python wrappers raise with the entry point and the reason."""
    fov = np.linspace(1.0, 1.2, 8)
    ts = np.arange(8) * (1000.0 / 30.0)
    with pytest.raises(g.GyroflowCoreError) as e:
        g.zoom_dynamic(fov, 1.0e7, 30.0, method=0)
    assert e.value.code == GF_ERR_BAD_PARAMS
    assert "gf_zoom_dynamic_compute: " in str(e.value) and "longer than" in str(e.value), str(e.value)
    with pytest.raises(g.GyroflowCoreError) as e:
        g.zoom_fovs(g.ZoomParams(1.0e7, method=0, scaled_fps=30.0), ts, fov)
    assert e.value.code == GF_ERR_BAD_PARAMS
    assert "gf_zoom_fovs: " in str(e.value) and "longer than" in str(e.value), str(e.value)
