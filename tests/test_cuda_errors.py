"""How the C ABI reports a failed CUDA call: the failure says why it happened and leaves nothing behind that fails the thread's
next call.  Every failing call here fails before anything is launched."""
import ctypes as C
import threading

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi, synth
from tests import cases, oracle_lib

pytestmark = pytest.mark.gpu


def test_failed_allocation_does_not_fail_the_next_frame():
    """A drawing buffer of 2^50 bytes: no host can page-lock that much, so its staging allocation fails before any byte of the drawing
    is read.  The next frame on the same context must render as if the failure had not happened."""
    p, src, m, mesh, dst0, pix, lens, digital = cases.build(dict(w=320, h=180))
    p.flags |= abi.FLAG_DRAWING_ENABLED
    want = dst0.copy()
    assert oracle_lib.undistort_image(src, want, p, pix, lens, digital, m, mesh) == 0
    got = dst0.copy()
    bufs = g.Buffers(g.BufferDescription((320, 180, p.stride), src), g.BufferDescription((320, 180, p.output_stride), got))
    w = g.CudaWrapper.new(p, pix, lens, digital, bufs)
    try:
        w.set_overlays(True)
        i, o = bufs.input.to_c(), bufs.output.to_c()
        mats = np.ascontiguousarray(m, dtype=np.float32)
        drawing = np.zeros(64, np.uint8)
        rc = w._lib.gf_cuda_undistort_image(w._h, C.byref(i), C.byref(o), C.byref(p), mats.ctypes.data, mats.shape[0], None, 0,
                                            drawing.ctypes.data, 2 ** 50, None)
        assert abi.ERRORS[rc] == "CudaError"
        assert w._lib.gf_cuda_last_error(w._h)
        # no drawing this time; the default safe area is the whole frame, so the overlays leave the frame as the oracle renders it
        w.undistort_image(bufs, g.FrameTransform(matrices=m, kernel_params=p))
        assert np.array_equal(got, want)
    finally:
        w.close()


def test_failed_gyro_upload_says_why():
    """A device index past the last device: the upload fails at cudaSetDevice and leaves the reason in gf_cuda_last_error(NULL)."""
    lib = g.load_library()
    cp = g.ComputeParams(synth.base_kernel_params(64, 36), *cases.gyro())
    result = {}

    def upload():                                   # on a fresh thread, whose last error starts out empty
        h = C.c_void_p()
        result["rc"] = lib.gf_cuda_gyro_upload(C.byref(h), lib.gf_cuda_device_count(), C.byref(cp.c))
        result["msg"] = lib.gf_cuda_last_error(None)

    t = threading.Thread(target=upload)
    t.start()
    t.join()
    assert abi.ERRORS[result["rc"]] == "CudaError"
    assert b"cudaErrorInvalidDevice" in result["msg"], result["msg"]
