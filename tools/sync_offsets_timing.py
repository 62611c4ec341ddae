#!/usr/bin/env python3
"""Wall time of the visual-features sync search on a synthetic 3840 x 2160 opencv_fisheye clip with rolling shutter.

  offsets : gf_cuda_find_sync_offsets, for_rs = 0 — the "Visual features" offset method (search_size candidates 1 ms apart, then 200
            candidates 0.01 ms apart, per range)
  rs      : gf_cuda_find_sync_offsets, for_rs = 1 — "Estimate rolling shutter" (2 * (1000 / fps) readout times, then 200)

The clip has --ranges ranges of --pairs matched pairs of --points points each (the second list moved by a few pixels plus noise).  Each
search is warmed up once and timed --reps times; the median wall time of the call (host clock around the synchronous call) is reported
with its host record time and device time (gf_cuda_sync_last_timing), next to one run of the CPU oracle (oracle/gf_oracle_sync.c) on all
host threads for the same job, and the card's name and power limit.  The device's chosen values are checked against the oracle's: with
the rotation on they may differ where the f64 slerp differs by an ulp, so the check is that the oracle's cost at the device's value is
within 0.1 % of the oracle's minimum.  Prints one JSON line (and writes it to --out if given).
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import gyroflow_b200 as g
from gyroflow_b200 import synth
from tests import oracle_lib
from tests.test_sync_offsets import oracle_costs, oracle_find


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
    ap.add_argument("--fps", type=float, default=30.0)
    ap.add_argument("--ranges", type=int, default=4)
    ap.add_argument("--pairs", type=int, default=8)
    ap.add_argument("--points", type=int, default=300)
    ap.add_argument("--search-size", type=float, default=200.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "no CUDA device: this script times the GPU"
    w, h, lens = a.width, a.height, "opencv_fisheye"
    p = synth.base_kernel_params(w, h, lens=lens)
    org, sm = synth.synthetic_gyro(4.0)
    cp = g.ComputeParams(p, org, sm, frame_readout_time_ms=16.0)
    dg = g.DeviceGyro(cp)
    rng = np.random.default_rng(11)
    ranges, span = [], 3_600_000 // a.ranges
    for r in range(a.ranges):
        pairs = []
        for i in range(a.pairs):
            ts = 200_000 + r * span + i * int(1e6 / a.fps) * 3
            p1 = (rng.random((a.points, 2)) * [0.8 * w, 0.8 * h] + [0.1 * w, 0.1 * h]).astype(np.float32)
            p2 = (p1 + np.float32([6.0, -3.0]) + rng.normal(0, 1.0, p1.shape)).astype(np.float32)
            pairs.append(((ts, p1), (ts + int(round(1e6 / a.fps)), p2)))
        ranges.append((200_000 + r * span, 200_000 + (r + 1) * span, pairs))
    searches = {"offsets": dict(initial_offset_ms=0.0, search_size_ms=a.search_size, for_rs=False),
                "rs": dict(for_rs=True)}
    result = dict(card=card(), size=[w, h], lens=lens, fps=a.fps, ranges=a.ranges, pairs_per_range=a.pairs, points_per_pair=a.points,
                  host_threads=oracle_lib.load().gf_oracle_online_cpus())
    for name, kw in searches.items():
        dev = dg.find_sync_offsets(lens, None, a.fps, ranges, **kw)          # warm-up
        walls, timings = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            dev = dg.find_sync_offsets(lens, None, a.fps, ranges, **kw)
            walls.append(time.perf_counter() - t0)
            timings.append(dg.sync_timing())
        k = int(np.argsort(walls)[len(walls) // 2])
        t0 = time.perf_counter()
        ora = oracle_find(cp, lens, None, ranges, kw.get("initial_offset_ms", 0.0), kw.get("search_size_ms", 0.0), kw["for_rs"], fps=a.fps)
        oracle_s = time.perf_counter() - t0
        agree = len(dev) == len(ora)
        mids = {(r0 + (r1 - r0) / 2.0) / 1000.0: pairs for r0, r1, pairs in ranges}
        for i, ((t, v, _), (_, _, c_min)) in enumerate(zip(dev, ora)):
            pairs = ranges[i][2] if kw["for_rs"] else mids[t]
            if kw["for_rs"]:
                c = oracle_costs(cp, lens, None, pairs, readouts=[v], clear=False, fps=a.fps)[0]
            else:
                c = oracle_costs(cp, lens, None, pairs, offsets=[v], fps=a.fps)[0]
            agree = agree and c <= c_min * 1.001
        n_cand = (int(a.search_size) if not kw["for_rs"] else 2 * int(1000.0 / a.fps)) + 200
        result[name] = dict(candidates_per_range=n_cand, call_ms=1e3 * walls[k], host_record_ms=timings[k]["host_record_ms"],
                            device_ms=timings[k]["device_ms"], chunks=timings[k]["chunks"], oracle_all_threads_ms=1e3 * oracle_s,
                            exact_match=dev == ora, agrees_with_oracle=bool(agree), results=dev)
    dg.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
