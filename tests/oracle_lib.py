"""ctypes access to the CPU oracle (oracle/libgf_oracle.so).  TESTS / smoke / cpu_baseline ONLY — never the product."""
import ctypes as C
import os
import subprocess

import numpy as np

from gyroflow_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE_DIR, "libgf_oracle.so")

_lib = None


def build():
    subprocess.check_call(["make", "-C", ORACLE_DIR, "-s"])


def load():
    global _lib
    if _lib is not None:
        return _lib
    src_m = max(os.path.getmtime(os.path.join(ORACLE_DIR, f)) for f in ("gf_oracle.c", "gf_oracle.h", "gf_coeffs.inc"))
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < src_m:
        build()
    lib = C.CDLL(LIB)
    P = C.POINTER
    lib.gf_oracle_undistort_image.restype = C.c_int
    lib.gf_oracle_undistort_image.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, P(abi.KernelParams), C.c_int, C.c_int, C.c_int,
                                              C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    lib.gf_oracle_lens_undistort_point.restype = C.c_int
    lib.gf_oracle_lens_undistort_point.argtypes = [C.c_int, C.c_float, C.c_float, P(abi.KernelParams), P(C.c_float), P(C.c_float)]
    lib.gf_oracle_lens_distort_point.restype = None
    lib.gf_oracle_lens_distort_point.argtypes = [C.c_int, C.c_float, C.c_float, C.c_float, P(abi.KernelParams), P(C.c_float), P(C.c_float)]
    lib.gf_oracle_rotate_and_distort.restype = C.c_int
    lib.gf_oracle_rotate_and_distort.argtypes = [C.c_float, C.c_float, C.c_size_t, P(abi.KernelParams), C.c_void_p, C.c_int, C.c_int,
                                                 C.c_void_p, C.c_size_t, P(C.c_float), P(C.c_float)]
    lib.gf_oracle_undistort_coord.restype = C.c_int
    lib.gf_oracle_undistort_coord.argtypes = [C.c_float, C.c_float, P(abi.KernelParams), C.c_void_p, C.c_int, C.c_int,
                                              C.c_void_p, C.c_size_t, P(C.c_float), P(C.c_float)]
    lib.gf_oracle_interpolate_mesh.restype = None
    lib.gf_oracle_interpolate_mesh.argtypes = [C.c_double, C.c_double, C.c_void_p, P(C.c_double), P(C.c_double)]
    lib.gf_oracle_find_fov.restype = C.c_double
    lib.gf_oracle_find_fov.argtypes = [P(abi.ComputeParams), C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_double, C.c_size_t]
    lib.gf_oracle_undistort_points_rs_ex.restype = None
    lib.gf_oracle_undistort_points_rs_ex.argtypes = [P(abi.ComputeParams), C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_double, C.c_size_t, C.c_double, C.c_int, C.c_void_p]
    lib.gf_oracle_stmap_undistort.restype = None
    lib.gf_oracle_stmap_undistort.argtypes = [P(abi.KernelParams), C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.gf_oracle_stmap_distort.restype = None
    lib.gf_oracle_stmap_distort.argtypes = [P(abi.ComputeParams), C.c_int, C.c_int, C.c_double, C.c_size_t, C.c_void_p]
    lib.gf_oracle_undistort_points_rs.restype = None
    lib.gf_oracle_undistort_points_rs.argtypes = [P(abi.ComputeParams), C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_double, C.c_size_t, C.c_double, C.c_void_p]
    lib.gf_oracle_zoom_dynamic.restype = None
    lib.gf_oracle_zoom_dynamic.argtypes = [C.c_void_p, C.c_size_t, C.c_double, C.c_double, C.c_int, C.c_void_p]
    lib.gf_oracle_draw_overlays.restype = None
    lib.gf_oracle_draw_overlays.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, P(abi.KernelParams), C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    lib.gf_oracle_online_cpus.restype = C.c_int
    lib.gf_oracle_describe.restype = C.c_char_p
    _lib = lib
    return lib


def undistort_image(src, dst, params, pixel_type, lens, digital_lens, matrices, mesh=None, threads=0):
    """Run the oracle in place on `dst` (numpy uint8, C-contiguous).  Returns the oracle's status code."""
    lib = load()
    m = np.ascontiguousarray(matrices, dtype=np.float32)
    mesh = np.zeros(0, np.float32) if mesh is None else np.ascontiguousarray(mesh, dtype=np.float32)
    assert src.dtype == np.uint8 and dst.dtype == np.uint8 and src.flags["C_CONTIGUOUS"] and dst.flags["C_CONTIGUOUS"]
    return lib.gf_oracle_undistort_image(src.ctypes.data, src.nbytes, dst.ctypes.data, dst.nbytes, C.byref(params),
                                         abi.PIXEL_TYPES[pixel_type][0], abi.LENS[lens], abi.LENS[digital_lens] if digital_lens else 0,
                                         m.ctypes.data, m.shape[0], mesh.ctypes.data if mesh.size else None, mesh.size, threads)


def distort_point(lens, x, y, z, params):
    lib = load(); ox, oy = C.c_float(), C.c_float()
    lib.gf_oracle_lens_distort_point(abi.LENS[lens], x, y, z, C.byref(params), C.byref(ox), C.byref(oy))
    return ox.value, oy.value


def undistort_point(lens, x, y, params):
    lib = load(); ox, oy = C.c_float(), C.c_float()
    ok = lib.gf_oracle_lens_undistort_point(abi.LENS[lens], x, y, C.byref(params), C.byref(ox), C.byref(oy))
    return (ox.value, oy.value) if ok else None


def undistort_coord(x, y, params, matrices, lens, digital_lens, mesh=None):
    """undistort_coord of cpu_undistort.rs:421-517 for output buffer position (x, y) (float32): the source position in buffer
    coordinates, or None."""
    lib = load(); ou, ov = C.c_float(), C.c_float()
    m = np.ascontiguousarray(matrices, dtype=np.float32)
    mesh = np.zeros(0, np.float32) if mesh is None else np.ascontiguousarray(mesh, dtype=np.float32)
    ok = lib.gf_oracle_undistort_coord(float(x), float(y), C.byref(params), m.ctypes.data, abi.LENS[lens], abi.LENS[digital_lens] if digital_lens else 0,
                                       mesh.ctypes.data if mesh.size else None, mesh.size, C.byref(ou), C.byref(ov))
    return (np.float32(ou.value), np.float32(ov.value)) if ok else None


def find_fovs(cp, lens, digital_lens, timestamps_ms, margin=2.0):
    """FovIterative::compute with the calculate_fovs adjustments (zooming/mod.rs:41-49): oracle, one frame at a time."""
    lib = load()
    c = abi.ComputeParams()
    C.memmove(C.byref(c), C.byref(cp.c), C.sizeof(abi.ComputeParams))
    ow, oh = c.output_width, c.output_height
    c.fov_scale = 1.0; c.n_fovs = 0; c.n_minimal_fovs = 0; c.output_width = c.width; c.output_height = c.height
    return np.array([lib.gf_oracle_find_fov(C.byref(c), abi.LENS[lens], abi.LENS[digital_lens] if digital_lens else 0, ow, oh, margin, float(t), i)
                     for i, t in enumerate(timestamps_ms)])


def zoom_dynamic(fov_minimal, window_s, fps, method=1):
    lib = load()
    a = np.ascontiguousarray(fov_minimal, dtype=np.float64); out = np.zeros_like(a)
    lib.gf_oracle_zoom_dynamic(a.ctypes.data, a.size, window_s, fps, method, out.ctypes.data)
    return out


def draw_overlays(buf, width, height, stride, params, pixel_type, is_input, drawing):
    """draw_pixel / draw_safe_area of opencl_undistort.cl:109-154 in place on `buf` (oracle restatement)."""
    lib = load()
    d = np.ascontiguousarray(drawing if drawing is not None else np.zeros(0, np.uint8), dtype=np.uint8)
    lib.gf_oracle_draw_overlays(buf.ctypes.data, buf.nbytes, width, height, stride, C.byref(params), abi.PIXEL_TYPES[pixel_type][0], int(is_input),
                                d.ctypes.data if d.size else None, d.size)
