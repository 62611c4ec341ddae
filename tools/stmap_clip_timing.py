#!/usr/bin/env python3
"""Frames per second of a clip's ST-map export: a 3840 x 2160 clip of 64 frames, opencv_fisheye with rolling shutter, per_frame = 1.

  loop : gf_cuda_generate_stmap once per frame (size query, then the maps) into preallocated device buffers — what a caller does
         without the clip entry points; host clock from the first call to the end of the last (each call synchronises).
  job  : gf_cuda_stmap_sizes + gf_cuda_generate_stmaps_dev for the whole clip, CUDA events on the stream around both calls.

Both are warmed up once and timed --reps times; the median is reported, with the card's name and power limit.  The maps of both
paths are compared bit for bit on the last repetition.  Prints one JSON line (and writes it to --out if given).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import gyroflow_b200 as g
from gyroflow_b200 import abi, synth


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:          # the number still stands; say why the card line is missing
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "no CUDA device: this script times the GPU"
    w, h, n = a.width, a.height, a.frames
    p = synth.base_kernel_params(w, h, lens="opencv_fisheye")
    org, sm = synth.synthetic_gyro(4.0)
    cp = g.ComputeParams(p, org, sm, frame_readout_time_ms=16.0)
    dg = g.DeviceGyro(cp)
    lib, m = dg._lib, abi.LENS["opencv_fisheye"]
    frames = np.arange(n, dtype=np.uintp)
    ts = (np.arange(n) * (1000.0 / 30.0) + 50.0).astype(np.float64)
    stream = torch.cuda.current_stream()
    st = stream.cuda_stream or 1                 # cudaStreamLegacy: NULL would mean the gyro object's own stream

    nw, nh = dg.stmap_sizes("opencv_fisheye", None, ts, frames, True, st)
    cap = 3 * int((nw.astype(np.int64) * nh).max())
    dist = [torch.empty(w * h * 3, dtype=torch.float32, device="cuda") for _ in range(n)]
    und = [torch.empty(cap, dtype=torch.float32, device="cuda") for _ in range(n)]
    loop_d = [torch.empty(w * h * 3, dtype=torch.float32, device="cuda") for _ in range(n)]
    loop_u = [torch.empty(cap, dtype=torch.float32, device="cuda") for _ in range(n)]
    dp = (C.c_void_p * n)(*[t.data_ptr() for t in dist]); up = (C.c_void_p * n)(*[t.data_ptr() for t in und])
    cw, ch = C.c_int32(), C.c_int32()

    def loop():
        for i in range(n):
            rc = lib.gf_cuda_generate_stmap(dg._h, C.byref(cp.c), m, 0, 1, int(frames[i]), float(ts[i]), C.byref(cw), C.byref(ch), None, 0, None, 0, st)
            assert rc == 0, rc
            rc = lib.gf_cuda_generate_stmap(dg._h, C.byref(cp.c), m, 0, 1, int(frames[i]), float(ts[i]), C.byref(cw), C.byref(ch),
                                            loop_d[i].data_ptr(), w * h * 3, loop_u[i].data_ptr(), cap, st)
            assert rc == 0, rc

    def job():
        sw, sh = np.zeros(n, np.int32), np.zeros(n, np.int32)
        rc = lib.gf_cuda_stmap_sizes(dg._h, C.byref(cp.c), m, 0, 1, frames.ctypes.data, ts.ctypes.data, n, sw.ctypes.data, sh.ctypes.data, st)
        assert rc == 0, rc
        rc = lib.gf_cuda_generate_stmaps_dev(dg._h, C.byref(cp.c), m, 0, 1, frames.ctypes.data, ts.ctypes.data, n, sw.ctypes.data, sh.ctypes.data,
                                             dp, up, w * h * 3, cap, st)
        assert rc == 0, rc

    loop(); job(); torch.cuda.synchronize()          # warm-up: module loads, the job's warp context, allocator
    t_loop, t_job = [], []
    for _ in range(a.reps):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        loop()
        torch.cuda.synchronize(); t_loop.append(time.perf_counter() - t0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream); job(); e1.record(stream)
        e1.synchronize(); t_job.append(e0.elapsed_time(e1) / 1000.0)
    same = all(torch.equal(loop_d[i].view(torch.int32), dist[i].view(torch.int32)) and
               torch.equal(loop_u[i][: 3 * int(nw[i]) * int(nh[i])].view(torch.int32), und[i][: 3 * int(nw[i]) * int(nh[i])].view(torch.int32))
               for i in range(n))
    dg.close()
    res = dict(card=card(), width=w, height=h, frames=n, lens="opencv_fisheye", rolling_shutter=True, per_frame=1,
               new_size_max=[int(nw.max()), int(nh.max())], reps=a.reps,
               loop_s=[round(x, 4) for x in t_loop], job_s=[round(x, 4) for x in t_job],
               loop_fps=round(n / float(np.median(t_loop)), 2), job_fps=round(n / float(np.median(t_job)), 2), maps_identical=bool(same))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    assert same, "the clip job's maps differ from the per-frame loop's"


if __name__ == "__main__":
    main()
