"""gyroflow_b200 — H100 (sm_90a) backend for Gyroflow's per-pixel stabilization warp.

Product code = gyroflow_b200/csrc (CUDA kernels + extern "C" ABI, built into libgyroflow_cuda.so).
This package is the thin host-side mirror used by tests and bench.py.
"""
from . import abi
from .abi import KernelParams, BackendMissing, load_library
from .backend import (BufferDescription, Buffers, FrameTransform, ProcessedInfo, CudaWrapper,
                      GyroflowCoreError, list_devices, ComputeParams, DeviceGyro, zoom_dynamic,
                      ZoomParams, zoom_fovs, scan_tables_dev, bind_thread_to_device, stab_config, get_frame_transform_at, host_register, host_unregister,
                      selftest_sync_select, optimal_sync_sizes, optimal_sync_select, optimal_sync_points, get_optimal_sync_points,
                      selftest_optimal_sync_resample)
from .render_queue import RenderQueue

__all__ = ["abi", "KernelParams", "BackendMissing", "load_library", "BufferDescription", "Buffers", "FrameTransform",
           "ProcessedInfo", "CudaWrapper", "GyroflowCoreError", "list_devices", "ComputeParams", "DeviceGyro", "zoom_dynamic",
           "ZoomParams", "zoom_fovs", "scan_tables_dev", "bind_thread_to_device", "stab_config", "get_frame_transform_at", "RenderQueue", "host_register", "host_unregister",
           "selftest_sync_select", "optimal_sync_sizes", "optimal_sync_select", "optimal_sync_points", "get_optimal_sync_points",
           "selftest_optimal_sync_resample"]
